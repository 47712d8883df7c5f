"""The angular count bound of the pruned v3 vote (csrc/prune.cu, DESIGN.md 4.2) against the oracle's exact counts.

A numpy twin of prune_hist_kernel + count_bound (float32 like the kernels) must give B(h) >= count(h) for every hypothesis:
the pruned vote skips exactly the hypotheses with B(h) below an exact count, so a bound below a count could change the
winner.  Bench shapes at small B, four thresholds, and inputs built to sit on the bound's edges."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import pvnet_oracle as po  # noqa: E402
from clean_pvnet_b200 import synth  # noqa: E402

TILE, NBIN = 1024, 64            # PRUNE_TILE, PRUNE_NBIN (csrc/kernels.h)
EPS = np.float32(1e-5)
F = np.float32


def prune_rotation(t):
    """prune_setup: (cos, sin) of theta' rounded outward, or None where nothing can be pruned."""
    t = float(np.float32(t))
    if not (0.0 < t < 1.0):
        return None
    w = math.acos(max(-1.0, t - 64.0 * 2.0 ** -24)) + 1e-5
    if not w < 1.5:
        return None
    return np.nextafter(F(math.cos(w)), F(0)), np.nextafter(F(math.sin(w)), F(1))


def pseudo_angle(x, y):
    x, y = np.asarray(x, F), np.asarray(y, F)
    with np.errstate(all="ignore"):
        p = np.where(y >= 0, np.where(x >= 0, y / (x + y), F(1) + (-x) / (y - x)),
                     np.where(x < 0, F(2) + (-y) / (-x - y), F(3) + x / (x - y)))
    return p.astype(F)


def tile_records(xy, dirs):
    """prune_hist_kernel for one (image, keypoint): [(box (x0,x1,y0,y1), inclusive prefix counts [NBIN])]"""
    recs = []
    for t0 in range(0, len(xy), TILE):
        c, v = xy[t0:t0 + TILE], dirs[t0:t0 + TILE]
        with np.errstate(all="ignore"):
            n1 = np.sqrt((v[:, 0].astype(np.float64) * v[:, 0] + v[:, 1].astype(np.float64) * v[:, 1]).astype(F))
        ok = (n1 > F(1e-6)) & (n1 < np.inf)
        bins = np.minimum(NBIN - 1, (pseudo_angle(v[ok, 0], v[ok, 1]) * F(NBIN // 4)).astype(np.int64))
        recs.append(((c[:, 0].min(), c[:, 0].max(), c[:, 1].min(), c[:, 1].max()),
                     np.cumsum(np.bincount(bins, minlength=NBIN))))
    return recs


def count_bound(hyp, recs, tn, rot):
    """count_bound for every hypothesis [hn,2]; tn for all when rot is None (nothing pruned)"""
    hx, hy = hyp[:, 0].astype(F), hyp[:, 1].astype(F)
    if rot is None:
        return np.full(len(hyp), tn, np.int64)
    c, s = rot
    out = np.zeros(len(hyp), np.int64)
    with np.errstate(all="ignore"):
        big = ~(np.abs(hx) + np.abs(hy) <= F(1e15))
        for (x0, x1, y0, y1), P in recs:
            tot = int(P[-1])
            inside = (hx >= x0 - F(0.5)) & (hx <= x1 + F(0.5)) & (hy >= y0 - F(0.5)) & (hy <= y1 + F(0.5))
            lx, ly = hx - x0, hy - y0
            ux, uy = lx.copy(), ly.copy()
            for cx, cy in ((x1, y0), (x0, y1), (x1, y1)):
                dx, dy = hx - F(cx), hy - F(cy)
                m = lx * dy - ly * dx < 0
                lx, ly = np.where(m, dx, lx), np.where(m, dy, ly)
                m = ux * dy - uy * dx > 0
                ux, uy = np.where(m, dx, ux), np.where(m, dy, uy)
            plo = pseudo_angle(c * lx + s * ly, c * ly - s * lx)
            phi = pseudo_angle(c * ux - s * uy, c * uy + s * ux)
            phi = np.where(phi < plo, phi + F(4), phi)
            blo = np.floor((plo - EPS) * F(NBIN // 4)).astype(np.int64)
            bhi = np.floor((phi + EPS) * F(NBIN // 4)).astype(np.int64)
            Pex = np.concatenate([[0], P])

            def C(j):
                w = np.floor_divide(j, NBIN)
                return Pex[j - w * NBIN] + tot * w
            part = np.where(bhi - blo + 1 >= NBIN, tot, C(bhi + 1) - C(blo))
            out += np.where(inside, tot, part)
    out[big] = tn
    return out


def _check(xy, dirs, hyp, t):
    """B(h) >= the oracle's count for every hypothesis; returns the fraction a winner count would exclude"""
    cnt = po.vote_count(dirs[:, None, :], xy, hyp[:, None, :], t)[:, 0]
    bnd = count_bound(hyp, tile_records(xy, dirs), len(xy), prune_rotation(t))
    bad = np.nonzero(bnd < cnt)[0]
    assert bad.size == 0, f"bound below count at t={t}: h={hyp[bad[:3]]} bound={bnd[bad[:3]]} count={cnt[bad[:3]]}"
    return float(np.mean(bnd < cnt.max())) if len(cnt) else 0.0


def _layer_case(cfg, B, t, seed):
    mask, vertex, _ = synth.make_inputs(cfg, device="cpu", seed=seed, B=B)
    m, v = mask.numpy(), vertex.numpy()
    hn = synth.CONFIGS[cfg]["hn"]
    _, dbg = po.ransac_voting_layer_v3(m, v, hn, inlier_thresh=t, seed=seed, debug=True)
    sel = po.select_pixels(m, mode=0, seed=seed)
    H, W = m.shape[1:]
    excluded = []
    for b in range(B):
        pix = sel["pix"][b]
        if len(pix) == 0:
            continue
        xy = np.stack([pix % W, pix // W], 1).astype(F)
        for k in range(v.shape[3]):
            dirs = v[b, pix // W, pix % W, k].astype(F)
            hyp = dbg["hyp"][b, k].astype(F)
            bnd = count_bound(hyp, tile_records(xy, dirs), len(pix), prune_rotation(t))
            cnt = dbg["counts"][b, k]
            assert np.all(bnd >= cnt), (cfg, b, k, t)
            excluded.append(np.mean(bnd < cnt.max()))
    return np.array(excluded)


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_bound_cfg1(t):
    _layer_case("cfg1", 1, t, 11)


@pytest.mark.parametrize("cfg,B", [("cfg2", 1), ("cfg3", 2), ("cfg5", 2)])
@pytest.mark.parametrize("t", [0.9, 0.99])
def test_bound_production_shapes(cfg, B, t):
    ex = _layer_case(cfg, B, t, 1236)
    if cfg == "cfg2" and t == 0.99:
        assert ex.mean() > 0.25          # the bound does exclude hypotheses on the bench workload


@pytest.mark.parametrize("t", [0.5, 0.999])
def test_bound_cfg2_extreme_thresholds(t):
    _layer_case("cfg2", 1, t, 77)


def _field(xy, kp, rng, noise=0.02):
    d = kp[None, :] - xy
    a = np.arctan2(d[:, 1], d[:, 0]) + rng.normal(0, noise, len(xy))
    return np.stack([np.cos(a), np.sin(a)], 1).astype(F)


def _near(h, rng, n):
    """points within a few ulps of h, and h itself"""
    out = [h]
    for _ in range(n):
        out.append([np.nextafter(F(h[0]), F(np.inf) if rng.random() < 0.5 else F(-np.inf)),
                    np.nextafter(F(h[1]), F(np.inf) if rng.random() < 0.5 else F(-np.inf))])
    return np.array(out, F)


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_bound_adversarial(t):
    rng = np.random.default_rng(5)
    # two tiles of a 48 x 45 block (the second one partly filled): corners, edges, just outside, pixels
    ys, xs = np.mgrid[10:58, 20:65]
    xy = np.stack([xs.ravel(), ys.ravel()], 1).astype(F)[:1500]
    dirs = _field(xy, np.array([40.0, 30.0]), rng)
    hyp = [[20, 10], [64, 10], [20, 31], [64, 31], [19.5, 10], [19.49, 5], [64.51, 31.49], [42, 9.49], [42, 31.51],
           [30, 60], [200, 12], [-100, -100], [40, 30], [1e6, 3], [3, -1e7], [1e16, 0], [np.nan, 4], [np.inf, 1]]
    for h in ([20, 10], [44, 31], [21, 32], [64, 41]):
        hyp.extend(_near(h, rng, 6))
    hyp = np.array(hyp, F)
    hyp = np.concatenate([hyp, (xy[rng.integers(0, len(xy), 40)] + rng.normal(0, 1e-5, (40, 2))).astype(F)])
    _check(xy, dirs, hyp, t)
    # votes aimed exactly at each hypothesis family, so counts are large where the bound is tight
    for aim in ([19.49, 5], [42, 31.51], [200, 12]):
        _check(xy, _field(xy, np.array(aim), rng, noise=0.0), hyp, t)


@pytest.mark.parametrize("t", [0.9, 0.99])
def test_bound_degenerate_tiles(t):
    rng = np.random.default_rng(6)
    # one-pixel tile, collinear tiles (a row and a column), repeated position
    for xy in (np.array([[7, 9]], F),
               np.stack([np.arange(0, 1300), np.full(1300, 5)], 1).astype(F),
               np.stack([np.full(1100, 3), np.arange(0, 1100)], 1).astype(F),
               np.tile(np.array([[4, 4]], F), (50, 1))):
        hyp = np.concatenate([xy[rng.integers(0, len(xy), 20)] + rng.normal(0, 2, (20, 2)),
                              [[7, 9], [7.5, 9], [6.49, 9], [-3, 5], [1400, 5], [3, -2], [3, 1200], [4, 4], [4.5, 3.5]],
                              rng.uniform(-50, 1400, (60, 2))]).astype(F)
        for aim in hyp[::7]:
            _check(xy, _field(xy, aim.astype(np.float64), rng, noise=0.01), hyp, t)


def test_bound_keypoint_outside_and_bad_vectors():
    rng = np.random.default_rng(7)
    ys, xs = np.mgrid[100:160, 200:300]
    xy = np.stack([xs.ravel(), ys.ravel()], 1).astype(F)
    kp = np.array([900.0, 130.0])                      # far outside the image
    dirs = _field(xy, kp, rng, noise=0.01)
    dirs[::7] = 0.0                                    # zero vectors never vote
    dirs[3::11] = np.nan                               # NaN vectors never vote
    dirs[5::13] *= F(1e-7)                             # below the norm cut
    dirs[6::17] *= F(1e30)                             # norm overflows
    hyp = np.concatenate([kp[None] + rng.normal(0, 3, (60, 2)), rng.uniform(0, 1000, (100, 2))]).astype(F)
    for t in (0.5, 0.9, 0.99, 0.999):
        _check(xy, dirs, hyp, t)


def test_bound_random_field_excludes_nothing():
    """Directions uniform at random: every tile's window holds about the whole tile, nothing can be excluded, and the
    bound must still hold."""
    rng = np.random.default_rng(8)
    ys, xs = np.mgrid[0:64, 0:64]
    xy = np.stack([xs.ravel(), ys.ravel()], 1).astype(F)
    a = rng.uniform(0, 2 * np.pi, len(xy))
    dirs = np.stack([np.cos(a), np.sin(a)], 1).astype(F)
    hyp = rng.uniform(-10, 74, (256, 2)).astype(F)
    assert _check(xy, dirs, hyp, 0.9) == 0.0


def test_no_pruning_outside_the_analysis():
    assert prune_rotation(0.0) is None and prune_rotation(1.0) is None and prune_rotation(-0.5) is None
    assert prune_rotation(0.05) is None                 # theta' >= 1.5
    assert prune_rotation(0.99) is not None
