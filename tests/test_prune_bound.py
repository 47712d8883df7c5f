"""The cell records and count bound of the pruned v3 vote (csrc/prune.cu, DESIGN.md 4.2) against the oracle's exact counts.

The bound is summed over the 32x32-pixel cells of the image.  The numpy twin in prune_twin.py must give B(h) >= the
oracle's count for every hypothesis: the pruned vote skips exactly the hypotheses whose bound is below an exact count, so
a bound below a count could change the winner.  Production shapes at four thresholds, inputs built on the cell borders and
on the bound's edges, degenerate cells and bad vectors; and where prune_setup turns pruning off."""
import numpy as np
import pytest

import pvnet_oracle as po
from clean_pvnet_b200 import synth
from prune_twin import F, cell_records, count_bound, field, near, prune_applies, prune_rotation, scored


def _check(xy, dirs, hyp, t, H, W):
    """B(h) >= the oracle's count for every hypothesis; returns the fraction a winner count would exclude"""
    cnt = po.vote_count(dirs[:, None, :], xy, hyp[:, None, :], t)[:, 0]
    bnd = count_bound(hyp, cell_records(xy, dirs, H, W), len(xy), prune_rotation(t))
    bad = np.nonzero(bnd < cnt)[0]
    assert bad.size == 0, f"bound below count at t={t}: h={hyp[bad[:3]]} bound={bnd[bad[:3]]} count={cnt[bad[:3]]}"
    return float(np.mean(bnd < cnt.max())) if len(cnt) else 0.0


def _layer_case(cfg, B, t, seed):
    """B(h) >= count(h) for every (image, keypoint, hypothesis); returns the excluded and the scored fraction per
    (image, keypoint)"""
    mask, vertex, _ = synth.make_inputs(cfg, device="cpu", seed=seed, B=B)
    m, v = mask.numpy(), vertex.numpy()
    hn = synth.CONFIGS[cfg]["hn"]
    _, dbg = po.ransac_voting_layer_v3(m, v, hn, inlier_thresh=t, seed=seed, debug=True)
    sel = po.select_pixels(m, mode=0, seed=seed)
    H, W = m.shape[1:]
    excluded, frac = [], []
    for b in range(B):
        pix = sel["pix"][b]
        if len(pix) == 0:
            continue
        xy = np.stack([pix % W, pix // W], 1).astype(F)
        for k in range(v.shape[3]):
            rec = cell_records(xy, v[b, pix // W, pix % W, k].astype(F), H, W)
            bnd = count_bound(dbg["hyp"][b, k].astype(F), rec, len(pix), prune_rotation(t))
            cnt = dbg["counts"][b, k]
            assert np.all(bnd >= cnt), (cfg, b, k, t)
            excluded.append(np.mean(bnd < cnt.max()))
            frac.append(scored(bnd, cnt) / hn)
    return np.array(excluded), np.array(frac)


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_bound_cfg1(t):
    _layer_case("cfg1", 1, t, 11)


@pytest.mark.parametrize("cfg,B", [("cfg2", 1), ("cfg3", 2), ("cfg4", 1), ("cfg5", 2)])
@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_cell_bound_production_shapes(cfg, B, t):
    """Two images on cfg3 and cfg5: synth's first image does not depend on B, so B = 2 covers B = 1 as well."""
    excluded, _ = _layer_case(cfg, B, t, 1236)
    if cfg == "cfg2" and t == 0.99:
        assert excluded.mean() > 0.25     # the bound does exclude hypotheses on the bench workload


def test_cell_bound_scores_under_045_on_cfg2():
    _, frac = _layer_case("cfg2", 2, 0.99, 1236)
    assert frac.mean() <= 0.45, frac.mean()


@pytest.mark.parametrize("t", [0.5, 0.999])
def test_bound_cfg2_extreme_thresholds(t):
    _layer_case("cfg2", 1, t, 77)


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_bound_adversarial(t):
    """A 48 x 45 block of a 64 x 70 image (the last row partly filled), straddling the cell borders x = 32 and 64 and
    y = 32: hypotheses on its corners and edges, just outside it, within ulps of pixels, and far away or non-finite."""
    rng = np.random.default_rng(5)
    H, W = 64, 70
    ys, xs = np.mgrid[10:58, 20:65]
    xy = np.stack([xs.ravel(), ys.ravel()], 1).astype(F)[:1500]
    dirs = field(xy, np.array([40.0, 30.0]), rng)
    hyp = [[20, 10], [64, 10], [20, 31], [64, 31], [19.5, 10], [19.49, 5], [64.51, 31.49], [42, 9.49], [42, 31.51],
           [30, 60], [200, 12], [-100, -100], [40, 30], [1e6, 3], [3, -1e7], [1e16, 0], [np.nan, 4], [np.inf, 1]]
    for h in ([20, 10], [44, 31], [21, 32], [64, 41]):
        hyp.extend(near(h, rng, 6))
    hyp = np.array(hyp, F)
    hyp = np.concatenate([hyp, (xy[rng.integers(0, len(xy), 40)] + rng.normal(0, 1e-5, (40, 2))).astype(F)])
    _check(xy, dirs, hyp, t, H, W)
    # votes aimed exactly at each hypothesis family, so counts are large where the bound is tight
    for aim in ([19.49, 5], [42, 31.51], [200, 12]):
        _check(xy, field(xy, np.array(aim), rng, noise=0.0), hyp, t, H, W)


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_cell_bound_adversarial(t):
    """A 75 x 101 image (neither side a multiple of 32): a block straddling the cell borders x = 31/32, 63/64 and
    y = 31/32, single-pixel cells, cells whose every vector is zero, NaN or below the norm cut, and hypotheses inside the
    boxes, within half a pixel of them and on the cell corners."""
    rng = np.random.default_rng(15)
    H, W = 75, 101
    ys, xs = np.mgrid[24:40, 26:70]
    pts = [np.stack([xs.ravel(), ys.ravel()], 1)]
    pts.append(np.array([[5, 5], [100, 3], [3, 74], [100, 74], [31, 70], [32, 70], [96, 64]]))   # single-pixel cells
    pts.append(np.stack(np.meshgrid(np.arange(66, 70), np.arange(66, 70)), -1).reshape(-1, 2))  # all-zero cell
    pts.append(np.stack(np.meshgrid(np.arange(70, 74), np.arange(45, 48)), -1).reshape(-1, 2))  # all-NaN cell
    pts.append(np.stack(np.meshgrid(np.arange(10, 14), np.arange(40, 44)), -1).reshape(-1, 2))  # below the norm cut
    xy = np.concatenate(pts).astype(F)
    order = np.lexsort((xy[:, 0], xy[:, 1]))             # raster order, as the selected-pixel list
    groups = np.concatenate([np.full(len(p), i) for i, p in enumerate(pts)])[order]
    xy = xy[order]
    hyp = [[26, 24], [69, 39], [31, 31], [32, 32], [31.5, 31.5], [32, 31], [31, 32], [63.5, 31.5], [64, 32],
           [25.5, 24], [25.49, 24], [69.51, 39.49], [45, 23.5], [45, 23.49], [45, 40.49], [5, 5], [5.5, 5.5], [5.51, 5],
           [96, 96], [0, 0], [32, 0], [0, 32], [64, 64], [96, 32], [100.5, 74.5], [50, 200], [-40, 30], [1e6, 3],
           [np.nan, 4], [np.inf, 1], [1e16, 0]]
    hyp = np.concatenate([np.array(hyp, F), rng.uniform(-20, 120, (60, 2)).astype(F)])
    for aim in ([31.5, 31.5], [25.49, 24], [64, 32], [5.51, 5], [50, 200]):
        dirs = field(xy, np.array(aim), rng, noise=0.0 if aim[0] == 64 else 0.01)
        dirs[groups == 2] = 0.0
        dirs[groups == 3] = np.nan
        dirs[groups == 4] *= F(1e-7)
        _check(xy, dirs, hyp, t, H, W)
        rec = cell_records(xy, dirs, H, W)
        tot = rec[:, -1].astype(np.int64) >> 16
        assert tot.sum() == np.count_nonzero(groups < 2)  # the zero, NaN and tiny vectors are in no cell


@pytest.mark.parametrize("t", [0.9, 0.99])
def test_bound_degenerate_cells(t):
    """A one-pixel cell, a one-row line across 41 cells, a one-column line across 35 cells, and 50 copies of one
    position, in an 1100 x 1300 image."""
    rng = np.random.default_rng(6)
    H, W = 1100, 1300
    for xy in (np.array([[7, 9]], F),
               np.stack([np.arange(0, 1300), np.full(1300, 5)], 1).astype(F),
               np.stack([np.full(1100, 3), np.arange(0, 1100)], 1).astype(F),
               np.tile(np.array([[4, 4]], F), (50, 1))):
        hyp = np.concatenate([xy[rng.integers(0, len(xy), 20)] + rng.normal(0, 2, (20, 2)),
                              [[7, 9], [7.5, 9], [6.49, 9], [-3, 5], [1400, 5], [3, -2], [3, 1200], [4, 4], [4.5, 3.5]],
                              rng.uniform(-50, 1400, (60, 2))]).astype(F)
        for aim in hyp[::7]:
            _check(xy, field(xy, aim.astype(np.float64), rng, noise=0.01), hyp, t, H, W)


def test_bound_keypoint_outside_and_bad_vectors():
    rng = np.random.default_rng(7)
    H, W = 480, 640
    ys, xs = np.mgrid[100:160, 200:300]
    xy = np.stack([xs.ravel(), ys.ravel()], 1).astype(F)
    kp = np.array([900.0, 130.0])                      # far outside the image
    dirs = field(xy, kp, rng, noise=0.01)
    dirs[::7] = 0.0                                    # zero vectors never vote
    dirs[3::11] = np.nan                               # NaN vectors never vote
    dirs[5::13] *= F(1e-7)                             # below the norm cut
    dirs[6::17] *= F(1e30)                             # norm overflows
    hyp = np.concatenate([kp[None] + rng.normal(0, 3, (60, 2)), rng.uniform(0, 1000, (100, 2))]).astype(F)
    for t in (0.5, 0.9, 0.99, 0.999):
        _check(xy, dirs, hyp, t, H, W)


def test_bound_random_field_excludes_nothing():
    """Directions uniform at random: every cell's window holds about the whole cell, nothing can be excluded, and the
    bound must still hold."""
    rng = np.random.default_rng(8)
    ys, xs = np.mgrid[0:64, 0:64]
    xy = np.stack([xs.ravel(), ys.ravel()], 1).astype(F)
    a = rng.uniform(0, 2 * np.pi, len(xy))
    dirs = np.stack([np.cos(a), np.sin(a)], 1).astype(F)
    hyp = rng.uniform(-10, 74, (256, 2)).astype(F)
    assert _check(xy, dirs, hyp, 0.9, 64, 64) == 0.0


def test_no_pruning_outside_the_analysis():
    assert prune_rotation(0.0) is None and prune_rotation(1.0) is None and prune_rotation(-0.5) is None
    assert prune_rotation(0.05) is None                 # theta' >= 1.5
    assert prune_rotation(0.99) is not None
    # prune_applies(t, hn, B, K): each condition of prune_setup on both sides of its edge
    for t in (0.0, 1.0, -0.5, 0.05):
        assert not prune_applies(t, 512, 4, 9), t
    assert prune_applies(0.08, 512, 4, 9) and prune_applies(0.99, 512, 4, 9)
    assert not prune_applies(0.99, 128, 4, 9)
    assert prune_applies(0.99, 129, 4, 9) and prune_applies(0.99, 2048, 4, 9)
    assert not prune_applies(0.99, 2049, 4, 9)
    assert not prune_applies(0.99, 512, 31, 1) and prune_applies(0.99, 512, 32, 1)
    assert not prune_applies(0.99, 2048, 1, 2048) and prune_applies(0.99, 2048, 1, 2047)   # pass 2's grid.y
