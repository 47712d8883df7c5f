"""The sub-cell records and the pass-2 refinement of the pruned v3 vote (csrc/prune.cu, DESIGN.md 4.2) on the CPU.

Pass 2 keeps a hypothesis only if B2(h), the count bound over the 16x16-pixel sub-cells, reaches pass 1's best count,
so B2(h) must be >= the oracle's count wherever B(h) must.  Every case of test_prune_bound.py runs again with the
sub-cell records in place of the cell records; then image sides on sub-cell borders, the cell record as the union of
its sub-cells, and how much the refinement removes on cfg-2."""
import numpy as np
import pytest

import pvnet_oracle as po
import test_prune_bound as tpb
from clean_pvnet_b200 import synth
from prune_subcell_twin import pass_lists, subcell_records
from prune_twin import CELL, REC, F, cell_records, count_bound, field, near, prune_rotation


@pytest.fixture
def subcells(monkeypatch):
    """test_prune_bound's checks, bounding over the sub-cell records"""
    monkeypatch.setattr(tpb, "cell_records", lambda xy, dirs, H, W: subcell_records(xy, dirs, H, W).reshape(-1, REC))


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_subcell_bound_cfg1(subcells, t):
    tpb.test_bound_cfg1(t)


@pytest.mark.parametrize("cfg,B", [("cfg2", 1), ("cfg3", 2), ("cfg4", 1), ("cfg5", 2)])
@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_subcell_bound_production_shapes(subcells, cfg, B, t):
    tpb._layer_case(cfg, B, t, 1236)


@pytest.mark.parametrize("t", [0.5, 0.999])
def test_subcell_bound_cfg2_extreme_thresholds(subcells, t):
    tpb.test_bound_cfg2_extreme_thresholds(t)


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_subcell_bound_adversarial(subcells, t):
    tpb.test_bound_adversarial(t)
    tpb.test_cell_bound_adversarial(t)


@pytest.mark.parametrize("t", [0.9, 0.99])
def test_subcell_bound_degenerate_cells(subcells, t):
    tpb.test_bound_degenerate_cells(t)


def test_subcell_bound_keypoint_outside_bad_vectors_and_random_field(subcells):
    tpb.test_bound_keypoint_outside_and_bad_vectors()
    tpb.test_bound_random_field_excludes_nothing()


def _union(sub):
    """the cell records formed from their sub-cells, as prune_hist_kernel forms them"""
    box = sub[:, :, :4].view(F)
    out = np.empty((len(sub), REC), np.int32)
    out[:, :4] = np.stack([box[:, :, 0].min(1), box[:, :, 1].max(1), box[:, :, 2].min(1), box[:, :, 3].max(1)],
                          1).view(np.int32)
    out[:, 4:] = sub[:, :, 4:].view("<u2").astype(np.int64).sum(1).astype("<u2").view(np.int32)
    return out


@pytest.mark.parametrize("H,W", [(49, 63), (50, 62), (47, 33), (64, 95), (61, 81)])
@pytest.mark.parametrize("t", [0.9, 0.99])
def test_subcell_borders(H, W, t):
    """Image sides that are 1..15 mod 16 (and sides on a cell border): a block straddling the sub-cell borders
    x = 15/16, 47/48 and y = 15/16, 31/32, the last partial row and column of sub-cells filled, hypotheses on the
    sub-cell corners and within ulps of them.  B and B2 hold, the cell record is the union of its sub-cells, and the
    sub-cells outside the image are empty."""
    rng = np.random.default_rng(H * 1000 + W)
    ys, xs = np.mgrid[10:min(H, 40), 12:min(W, 52)]
    pts = [np.stack([xs.ravel(), ys.ravel()], 1),
           np.stack(np.meshgrid(np.arange(W - 3, W), np.arange(H - 3, H)), -1).reshape(-1, 2),   # the last corner
           np.array([[15, 0], [16, 0], [0, 15], [0, 16], [W - 1, 0], [0, H - 1]])]
    xy = np.unique(np.concatenate(pts), axis=0)
    xy = xy[np.lexsort((xy[:, 0], xy[:, 1]))].astype(F)
    hyp = [[15, 15], [16, 16], [15.5, 15.5], [16, 15], [47, 31], [48, 32], [31.5, 15.5], [15.49, 10], [16.51, 10],
           [W, H], [W - 0.5, H - 0.5], [-5, 20], [200, 7], [np.nan, 1], [1e16, 0]]
    for h in ([16, 16], [48, 32], [W - 1, H - 1]):
        hyp.extend(near(h, rng, 4))
    hyp = np.concatenate([np.array(hyp, F), rng.uniform(-10, max(H, W) + 10, (60, 2)).astype(F)])
    rot = prune_rotation(t)
    for aim in ([16, 16], [15.49, 10], [48, 32], [W - 0.5, H - 0.5], [200, 7]):
        dirs = field(xy, np.array(aim), rng, noise=0.0 if aim[0] == 16 else 0.01)
        dirs[::9] = 0.0
        cnt = po.vote_count(dirs[:, None, :], xy, hyp[:, None, :], t)[:, 0]
        cells, sub = cell_records(xy, dirs, H, W), subcell_records(xy, dirs, H, W)
        b1 = count_bound(hyp, cells, len(xy), rot)
        b2 = count_bound(hyp, sub.reshape(-1, REC), len(xy), rot)
        assert (b1 >= cnt).all() and (b2 >= cnt).all(), (H, W, t, aim)
        assert np.array_equal(_union(sub), cells)
        ncx = (W + CELL - 1) // CELL
        for c in range(len(cells)):
            for j in range(4):
                x0, y0 = c % ncx * CELL + (j & 1) * 16, c // ncx * CELL + (j >> 1) * 16
                if x0 >= W or y0 >= H:
                    assert sub[c, j, -1] >> 16 == 0 and np.isinf(sub[c, j, :4].view(F)).all()


def test_subcells_cut_cfg2_pass_two():
    """On the bench workload (two images, t = 0.99) the refinement keeps the winners and removes most of pass 2
    (the twin gives 60 -> 14 entries per list over 16 images and three seeds)."""
    mask, vertex, _ = synth.make_inputs("cfg2", device="cpu", seed=1236, B=2)
    m, v = mask.numpy(), vertex.numpy()
    _, dbg = po.ransac_voting_layer_v3(m, v, 512, inlier_thresh=0.99, seed=1236, debug=True)
    sel = po.select_pixels(m, mode=0, seed=1236)
    H, W = m.shape[1:]
    coarse, fine = [], []
    for b in range(2):
        pix = sel["pix"][b]
        xy = np.stack([pix % W, pix // W], 1).astype(F)
        for k in range(v.shape[3]):
            d = v[b, pix // W, pix % W, k].astype(F)
            hyp, cnt = dbg["hyp"][b, k].astype(F), dbg["counts"][b, k]
            bnd = count_bound(hyp, cell_records(xy, d, H, W), len(pix), prune_rotation(0.99))
            b2 = count_bound(hyp, subcell_records(xy, d, H, W).reshape(-1, REC), len(pix), prune_rotation(0.99))
            assert (b2 >= cnt).all()
            p1, p2, p2_coarse = pass_lists(bnd, b2, cnt)
            assert np.argmax(cnt) in np.concatenate([p1, p2])
            coarse.append(len(p2_coarse))
            fine.append(len(p2))
    assert np.mean(fine) <= 0.5 * np.mean(coarse), (np.mean(fine), np.mean(coarse))
