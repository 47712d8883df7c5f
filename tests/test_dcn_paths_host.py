"""CPU tests of tests/dcn_paths.py: its twin of the half-precision forward's launch decisions restates csrc/dcn.cu's
constants, PATHS reaches every branch side it lists in both layouts and needs every one of its cases, and the fp64
restatement stays cheap at the largest case the GPU tests hand it."""
import os
import re

import numpy as np

import dcn_cases as dc
import dcn_oracle as do
import dcn_paths as dp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_the_twin_restates_the_kernel_constants():
    with open(os.path.join(ROOT, "clean_pvnet_b200", "csrc", "dcn.cu")) as f:
        src = f.read()
    consts = dict(re.findall(r"\b(H_TARGET_CTAS|H_MAX_SPLIT|H_MIN_CHUNKS|HBM|HBN|HBK|BN) = (\d+)", src))
    assert {k: int(v) for k, v in consts.items()} == dict(
        H_TARGET_CTAS=dp.H_TARGET_CTAS, H_MAX_SPLIT=dp.H_MAX_SPLIT, H_MIN_CHUNKS=dp.H_MIN_CHUNKS, HBM=dp.HBM,
        HBN=dp.HBN, HBK=dp.HBK, BN=dp.BN)


def test_the_twin_gives_the_splits_the_design_states_for_the_detector():
    """DESIGN.md section 8n: at 736x544 the 17x23 layer runs with S = 8, the 34x46 layers with S = 6 or 8, the 68x92
    layers with S = 3 and the 136x184 layers unsplit."""
    by_h = {}
    for c in dc.DETECTOR["544x736"]:
        by_h.setdefault(c.H, set()).add(dp.half_splits(c))
    assert by_h == {17: {8}, 34: {6, 8}, 68: {3}, 136: {1}}


def test_paths_are_small():
    for c in dp.PATHS:
        assert c.H <= 16 and c.W <= 16 and c.B <= 5, dc.case_id(c)


def test_paths_reach_every_cell_in_both_layouts():
    missing = dp.REQUIRED - dp.reached(dp.PATHS)
    assert not missing, sorted(missing)
    # what REQUIRED lists: the 16-byte and the scalar paths, every tail and split, and the partly filled output tiles
    names = {name for name, _ in dp.REQUIRED}
    assert {f"vec S={s}" for s in range(1, 9)} <= names
    assert {f"vec tail={t}" for t in (0, 8, 16, 24)} <= names
    assert {f"vec dg={g}" for g in (1, 2, 4)} <= names
    assert {c.Co for c in dp.PATHS if dp.vec(c)} >= {129, 200, 257}


def test_every_path_case_reaches_a_cell_no_other_case_does():
    """Dropping any one case from PATHS loses a cell, so an edit of the table cannot drop one silently."""
    for i, c in enumerate(dp.PATHS):
        rest = dp.PATHS[:i] + dp.PATHS[i + 1:]
        assert dp.REQUIRED - dp.reached(rest), dc.case_id(c)


def test_the_twin_sees_what_the_cells_name():
    """The twin's numbers for three PATHS cases, worked out by hand from dcn.cu."""
    c16 = dc.Case(2, 16, 7, 9, 200, 3, 3, (1, 1), (1, 1), (1, 1), 2)
    assert dp.vec(c16) and dp.tail(c16) == 8 and dp.half_splits(c16) == 4 and dp.otiles(c16) == 2
    assert dp.live_warps_in_last_tile(c16) == 3                # 72 channels in the second tile: rows 0-95 live
    assert dp.split_starts(c16) == [(0, 0, 0), (0, 4, 0), (1, 0, 0), (1, 4, 0)]
    c80 = dc.Case(2, 80, 8, 9, 72, 3, 3, (1, 1), (1, 1), (1, 1), 2)
    assert dp.nchunk(c80) == 36 and dp.half_splits(c80) == 8
    assert dp.split_starts(c80)[6] == (1, 4, 32)               # kb = 27: group 1, tap 4, its second chunk
    assert not dp.vec(dc.Case(2, 24, 7, 8, 20, 3, 3, (1, 1), (1, 1), (1, 1), 2))
    assert dp.grid(c80) == (16, 1, 2)


def test_backward_cases_reach_the_grad_weight_tiles_and_a_partial_chunk():
    tiles = {dp.grad_weight_tiles(c) for c in dp.BACKWARD}
    assert {(2, 8), (3, 1)} <= tiles
    for B in dp.BACKWARD_BATCHES:                              # chunks of 2 images: the last holds 1, at b0 = B - 1
        assert B % 2 == 1 and B > 2


def test_the_restatement_is_cheap_at_the_largest_case():
    """The GPU tests run dcn_oracle.forward and .backward on every PATHS case (backward also on GW_TILES) at up to 5
    images; at the largest the column matrix has under a million entries, and both run here."""
    big = max((c._replace(B=max(dp.BACKWARD_BATCHES)) for c in dp.BACKWARD), key=dp.column_entries)
    assert dp.column_entries(big) < 1 << 20
    x, off, m, w, b = dc.make_inputs(big, seed=0, offsets="random")
    out, out_abs = do.forward(x, off, m, w, b, big.stride, big.pad, big.dil, big.dg)
    go = np.ones_like(out, dtype=np.float32)
    r = do.backward(x, off, m, w, b, go, big.stride, big.pad, big.dil, big.dg)
    assert out.shape == (big.B, big.Co, *dc.out_hw(big)) and np.isfinite(out).all() and (out_abs >= 0).all()
    assert r["grad_weight"].shape == w.shape and np.isfinite(r["grad_input"]).all()
