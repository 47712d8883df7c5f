"""GPU: the pruned v3 vote (csrc/prune.cu) against the same call with every hypothesis scored (debug=True).

Bars: keypoints bit-identical, the same winner (point and first-max index), and for every hypothesis the pruned path
scored, the same count; the hypotheses it did not score have bounds below the winner's count and count 0.  Wherever
pruning runs (prune_twin.prune_applies), the cell records equal prune_twin.cell_records bit for bit, and on cfg-2 the two
passes score at most 0.45 of the hypotheses."""
import math

import numpy as np
import pytest
import torch

from prune_twin import CELL, REC, cell_records, prune_applies

pytestmark = pytest.mark.gpu

THRESH = 0.99


def _inputs(cfg, seed, **kw):
    from clean_pvnet_b200 import synth
    return synth.make_inputs(cfg, device="cuda", seed=seed, **kw)


def _pruned(pvb, mask, vertex, hn, thresh=THRESH, min_num=5, max_num=30000, **kw):
    """The plain (pruned) call, then its workspace: counts, hypotheses, the two pass lists and lengths, and the cell
    records."""
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    out = pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=thresh, min_num=min_num, max_num=max_num, **kw)
    torch.cuda.synchronize()
    lib = _lib.load()
    cap = kw.get("capacity") or (mask.shape[1] * mask.shape[2] if kw.get("selection") is not None else None)
    m, v = rv._check_inputs(mask, vertex)
    d = rv._make_desc(m, v, hn, thresh, min_num, max_num, _lib.PVB_SELECT_BYTE, kw.get("seed", 0), 0, cap)
    ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
    views = rv._views(ws, d, lib, refit=True)
    L = _lib.PvbLayout()
    _lib.check(lib.pvb_workspace_layout(d, L))
    B, K, H, W = d.B, d.K, d.H, d.W
    assert L.prune_ncells == math.ceil(H / CELL) * math.ceil(W / CELL)
    lists = ws[L.prune_list:L.prune_list + 2 * B * K * hn * 4].view(torch.int32).view(2, B, K, hn).cpu().numpy()
    lens = ws[L.prune_len:L.prune_len + 2 * B * K * 4].view(torch.int32).view(2, B, K).cpu().numpy()
    cells = ws[L.prune_cells:L.prune_cells + B * K * L.prune_ncells * REC * 4].view(torch.int32)
    cells = cells.view(B, K, L.prune_ncells, REC).cpu().numpy()
    return out, views, lists, lens, cells


def _first_max(c):
    return np.argmax(c, axis=-1)


def _compare(pvb, mask, vertex, hn, thresh=THRESH, **kw):
    """pruned == full, and where pruning runs the cell records equal the twin's (they are not written otherwise, and
    the workspace then holds stale ones); returns the fraction of hypotheses scored per (image, keypoint)"""
    out, views, lists, lens, cells = _pruned(pvb, mask, vertex, hn, thresh, **kw)
    full, dbg = pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=thresh, debug=True,
                                           min_num=kw.pop("min_num", 5), max_num=kw.pop("max_num", 30000), **kw)
    assert torch.equal(out.view(torch.int32), full.view(torch.int32)), "keypoints differ from the full path"
    assert torch.equal(views["hyp"].view(torch.int32), dbg["hyp"].view(torch.int32))
    assert torch.equal(views["win"].view(torch.int32), dbg["win"].view(torch.int32))
    cp, cf = views["counts"].cpu().numpy(), dbg["counts"].cpu().numpy()
    tn, state = dbg["tn"].cpu().numpy(), dbg["state"].cpu().numpy()
    B, K = cf.shape[:2]
    H, W = mask.shape[1:]
    xy, dirs = views["xy"].cpu().numpy(), views["dirs"].cpu().numpy()
    frac = np.ones((B, K))
    pruned = prune_applies(thresh, hn, B, K)
    for b in range(B):
        for k in range(K):
            if not pruned:
                assert np.array_equal(cp[b, k], cf[b, k])
                continue
            scored = np.zeros(hn, bool)
            for p in range(2):
                sel = lists[p, b, k, :lens[p, b, k]]
                assert len(np.unique(sel)) == len(sel) and (sel >= 0).all() and (sel < hn).all()
                assert not scored[sel].any(), "a hypothesis was scored twice"
                scored[sel] = True
            assert lens[0, b, k] == 128
            want = cell_records(xy[b, :tn[b]], dirs[b, k, :tn[b]], H, W)
            bad = np.nonzero((cells[b, k] != want).any(1))[0]
            assert bad.size == 0, f"image {b} keypoint {k}: cells {bad[:4]} differ from the twin"
            assert np.array_equal(cp[b, k][scored], cf[b, k][scored])
            assert (cp[b, k][~scored] == 0).all()
            if state[b] == 0 and tn[b] > 0:
                assert (cf[b, k][~scored] < cf[b, k].max()).all(), "an unscored hypothesis could win"
                assert _first_max(cp[b, k]) == _first_max(cf[b, k])
            frac[b, k] = scored.mean()
    return frac


@pytest.mark.parametrize("cfg,B", [("cfg2", 4), ("cfg3", 4), ("cfg4", 2), ("cfg5", 4)])
@pytest.mark.parametrize("layout", ["interleaved", "planar"])
def test_pruned_equals_full_baseline_shapes(pvb, cfg, B, layout):
    from clean_pvnet_b200 import synth
    mask, vertex, _ = _inputs(cfg, 1236, B=B, layout=layout)
    frac = _compare(pvb, mask, vertex, synth.CONFIGS[cfg]["hn"], seed=1000)
    if cfg == "cfg2":
        print(f"cfg2 scored fraction per (image, keypoint): mean {frac.mean():.3f} min {frac.min():.3f} max {frac.max():.3f}")
        assert frac.mean() <= 0.45


def test_pruned_cfg1_is_not_pruned(pvb):
    mask, vertex, _ = _inputs("cfg1", 3)
    _compare(pvb, mask, vertex, 64, seed=4)


@pytest.mark.parametrize("thresh", [0.5, 0.9, 0.999])
def test_pruned_thresholds(pvb, thresh):
    mask, vertex, _ = _inputs("cfg2", 21, B=4)
    _compare(pvb, mask, vertex, 512, thresh=thresh, seed=22)


def test_pruned_explicit_idxs_and_torch_rng(pvb):
    mask, vertex, _ = _inputs("cfg2", 31, B=4)
    B, H, W, K, _ = vertex.shape
    g = torch.Generator(device="cuda").manual_seed(3)
    idxs = torch.randint(0, 20000, (B, 512, K, 2), generator=g, device="cuda", dtype=torch.int32)
    _compare(pvb, mask, vertex, 512, idxs=idxs, seed=1)
    torch.manual_seed(9)
    a = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=THRESH, rng="torch")
    torch.manual_seed(9)
    b, _ = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=THRESH, rng="torch", debug=True)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("hn", [129, 256, 300, 1024, 1500, 2048, 2049])
def test_pruned_hypothesis_counts(pvb, hn):
    mask, vertex, _ = _inputs("small", 41, B=8)
    _compare(pvb, mask, vertex, hn, seed=42, max_num=900)


def test_pruned_skipped_images_and_small_tiles(pvb):
    mask, vertex, _ = _inputs("cfg2", 51, B=4)
    mask = mask.clone()
    mask[1] = 0                       # skipped image
    mask[2] = 0
    mask[2, 100:110, 200:230] = 1     # 300 pixels: fewer than one tile
    _compare(pvb, mask, vertex, 512, seed=52)


def test_pruned_nothing_votes_and_empty_pass_two(pvb):
    mask, vertex, _ = _inputs("cfg2", 61, B=4)
    # image 0: every vector zero -> every count 0, L = 0, nothing excluded (pass 2 scores the rest)
    v = vertex.clone()
    v[0] = 0.0
    frac = _compare(pvb, mask, v, 512, seed=62)
    assert (frac[0] == 1.0).all()
    # a noise-free field where 128 pairs give the keypoint and the other 384 pair a pixel with itself (hypothesis (0,0),
    # which hardly any pixel faces): pass 1 holds the winners, every other bound is below them -> pass 2 is empty
    m2, v2, _ = _inputs("cfg2", 63, B=4, noise_deg=0.0, outlier_frac=0.0)
    K = v2.shape[3]
    g = torch.Generator(device="cuda").manual_seed(65)
    idxs = torch.randint(0, 20000, (4, 512, K, 2), generator=g, device="cuda", dtype=torch.int32)
    idxs[:, 128:, :, 1] = idxs[:, 128:, :, 0]
    _, _, _, lens, _ = _pruned(pvb, m2, v2, 512, idxs=idxs, seed=64)
    assert (lens[1, 0] == 0).all()                    # image 0: every keypoint's pass 2 is empty
    _compare(pvb, m2, v2, 512, idxs=idxs, seed=64)


def test_pruned_host_buffer_and_decode_entries(pvb):
    mask, vertex, _ = _inputs("cfg2", 71, B=8)
    full, _ = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=THRESH, seed=72, debug=True)
    host = pvb.ransac_voting_layer_v3_host(mask.cpu().pin_memory(), vertex.cpu().pin_memory(), 512, inlier_thresh=THRESH,
                                           seed=72, chunk_images=4)
    assert torch.equal(host.view(torch.int32), full.cpu().view(torch.int32))
    # the fused decode (argmax of the logits in the select kernel) against the full path on the argmax mask
    from clean_pvnet_b200 import decode
    C = 3
    seg = torch.randn((8, C, mask.shape[1], mask.shape[2]), device="cuda")
    seg[:, 1] += mask.float() * 8
    want, _ = pvb.ransac_voting_layer_v3(torch.argmax(seg, 1), vertex, 512, inlier_thresh=THRESH, seed=73, debug=True)
    _, got = decode._decode_v3(seg, vertex, 512, THRESH, 5, 30000, 73, 0)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
