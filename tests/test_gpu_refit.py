"""GPU: the refit's inlier set under adversarial geometry.  The refit (refit_kernel in csrc/vote.cu) decides the winner's
inliers with its own fast prefilter, not with the vote kernel's verdicts, and its keypoint hides a wrong inlier set
(one pixel moves the solution by ~r/N).  Here the winner is forced -- every hypothesis is the same designed sample
pair, whose exact bits come from the oracle's generate_hypothesis -- and the debug `normal_eq` is compared with the sums
over the reference predicate's inliers (tests/util.py, rtol 1e-12), next to counts, winner and keypoint.

Designs: winner 1 ulp from a selected pixel (the reference's norm2 < 1e-6 cut) or exactly on it, pixels on the winner's
cone boundary at +-acos(t)*(1+-1e-7) from 0.5 to 1e5 px, direction norms {0, 1e-7, 1.1e-6, 1e4, 1e19, NaN, +-Inf}, the
prefilter's |d|_1 <= 1e6 limit, thresholds outside and inside (0,1), no winner at all, several 2048-pixel refit CTAs."""
import numpy as np
import pytest
import torch

from util import bits_equal, check_normal_eq, oracle_inliers

pytestmark = pytest.mark.gpu

f32 = np.float32


def _ulp_neighbours(x, n):
    """x and the n float32 neighbours on each side."""
    out, lo, hi = [f32(x)], f32(x), f32(x)
    for _ in range(n):
        lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
        out += [lo, hi]
    return np.array(out, dtype=f32)


def _near(v, ulp_t, lever, n):
    """Candidates for one direction component: its ulp neighbours, and steps that move the intersection by about an
    eighth of the target's ulp (`lever` = distance from the pixel to the target across that component)."""
    steps = np.float64(v) + np.arange(-n, n + 1) * (float(ulp_t) / (8.0 * max(lever, 1e-30)))
    return np.unique(np.concatenate([_ulp_neighbours(v, n), steps.astype(f32)]))


def _design_pair(oracle, A, B, target, exact=True, n=40):
    """Directions at pixels A and B whose ray intersection -- as the reference computes it -- is `target`, bit for bit
    when `exact`: the float32 unit vectors towards the target and small perturbations of one component of each are
    searched.  Returns (vA, vB, hypothesis)."""
    def towards(P):
        d = np.asarray(target, np.float64) - np.asarray(P, np.float64)
        return d / np.hypot(*d)
    a, b = towards(A), towards(B)
    tx, ty = f32(target[0]), f32(target[1])
    ax = _near(a[0], np.spacing(tx), abs(float(ty) - A[1]), n)
    by = _near(b[1], np.spacing(ty), abs(float(tx) - B[0]), n)
    cand = np.array([(x, y) for x in ax for y in by], dtype=f32)
    m = len(cand)
    direct = np.zeros((2 * m, 1, 2), dtype=f32)
    direct[0::2, 0] = np.stack([cand[:, 0], np.full(m, a[1], dtype=f32)], 1)
    direct[1::2, 0] = np.stack([np.full(m, b[0], dtype=f32), cand[:, 1]], 1)
    coords = np.zeros((2 * m, 2), dtype=f32)
    coords[0::2], coords[1::2] = A, B
    idxs = np.stack([np.arange(0, 2 * m, 2), np.arange(1, 2 * m, 2)], 1).astype(np.int32)[:, None, :]
    hyp = oracle.generate_hypothesis(direct, coords, idxs)[:, 0]
    t = np.asarray(target, dtype=f32)
    hit = np.flatnonzero((hyp == t).all(axis=1))
    if exact:
        assert hit.size, f"no sample pair at {A}, {B} meets {t.tolist()}"
        i = int(hit[0])
    else:
        i = int(np.argmin(np.abs(hyp.astype(np.float64) - np.asarray(target)).sum(axis=1)))
    return direct[2 * i, 0], direct[2 * i + 1, 0], hyp[i]


def _run(pvb, oracle, H, W, dirs, pairs, thresh, hn=8, mask=None):
    """One image: dirs [H,W,K,2] float32 at every pixel (selected: `mask`, default all), pairs[k] = ((xA,yA), (xB,yB)) the
    sample pair of every hypothesis of keypoint k.  Checks the layer against the oracle; returns (debug dict, keypoints)."""
    K = dirs.shape[2]
    if mask is None:
        mask = np.ones((H, W), dtype=np.uint8)
    order = np.full(H * W, -1, dtype=np.int64)
    sel = np.flatnonzero(mask.reshape(-1))
    order[sel] = np.arange(sel.size)                                # torch.nonzero order
    idxs = np.zeros((1, hn, K, 2), dtype=np.int32)
    for k, (A, B) in enumerate(pairs):
        idxs[0, :, k] = [order[A[1] * W + A[0]], order[B[1] * W + B[0]]]
    assert (idxs >= 0).all()
    m, v = mask[None].astype(np.int64), dirs[None].astype(f32)
    out, dbg = pvb.ransac_voting_layer_v3(torch.from_numpy(m).cuda(), torch.from_numpy(v).cuda(), hn,
                                          inlier_thresh=thresh, idxs=torch.from_numpy(idxs).cuda(), seed=0, debug=True)
    with np.errstate(all="ignore"):
        want, odbg = oracle.ransac_voting_layer_v3(m, v, hn, inlier_thresh=thresh, idxs=idxs, debug=True)
    assert np.array_equal(dbg["tn"].cpu().numpy(), odbg["tn"])
    assert bits_equal(dbg["hyp"].cpu().numpy(), odbg["hyp"])
    assert np.array_equal(dbg["counts"].cpu().numpy(), odbg["counts"])
    assert bits_equal(dbg["win"].cpu().numpy(), odbg["win"])
    check_normal_eq(dbg, thresh, oracle_inliers(oracle))
    got = out.cpu().numpy()
    # both solve the same float64 system; far keypoints are compared at a few float32 ulps
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    assert (np.abs(got[fin] - want[fin]) <= np.maximum(1e-4, 4e-7 * np.abs(want[fin]))).all()
    return dbg, got


def _towards(H, W, target, rng, noise_deg=4.0, outliers=0.2):
    """[H,W,2] float32 directions at every pixel towards `target` (noisy, some random): a consensus for the winner."""
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    ang = np.arctan2(target[1] - ys, target[0] - xs) + rng.normal(0, np.radians(noise_deg), (H, W))
    ang = np.where(rng.uniform(size=(H, W)) < outliers, rng.uniform(0, 2 * np.pi, (H, W)), ang)
    return np.stack([np.cos(ang), np.sin(ang)], -1).astype(f32)


# ---- winner within (0, 1e-6) of a selected pixel, or exactly on it ------------------------------------------------
_OFFSETS = [(1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, -1), (1, -1), (-1, 1), (0, 0)]


def _step(x, s):
    x = f32(x)
    return x if s == 0 else np.nextafter(x, f32(np.inf) if s > 0 else f32(-np.inf))


@pytest.mark.parametrize("thresh", [0.99, 0.5])
@pytest.mark.parametrize("cx,cy", [(3, 5), (0, 0), (1, 0), (0, 7), (2, 13), (8, 1), (15, 15), (7, 4), (12, 9), (1, 1)])
def test_winner_next_to_a_pixel(pvb, oracle, cx, cy, thresh):
    """Keypoint k's winner is pixel (cx, cy) moved by +-1 ulp in x, y or both, or the pixel itself.  Pixel coordinates
    0-15: only there is the float32 spacing fine enough for 0 < |h-c| < 1e-6.  The pixel points at the winner, so
    only the reference's norm cut rejects it."""
    H, W = 20, 20
    rng = np.random.default_rng(cx * 100 + cy)
    A = (cx, cy - 1 if cy > 0 else cy + 1)                 # neighbours in y and x: the sample pair
    B = (cx - 1 if cx > 0 else cx + 1, cy)
    dirs = np.zeros((H, W, len(_OFFSETS), 2), dtype=f32)
    pairs = []
    for k, (sx, sy) in enumerate(_OFFSETS):
        target = (_step(cx, sx), _step(cy, sy))
        dirs[:, :, k] = _towards(H, W, np.array(target, np.float64), rng)
        vA, vB, h = _design_pair(oracle, A, B, target)
        assert (h == np.array(target, dtype=f32)).all()              # (the sign of a zero may differ)
        dirs[A[1], A[0], k], dirs[B[1], B[0], k] = vA, vB
        d = np.array([sx, sy], np.float64)
        dirs[cy, cx, k] = (d / np.hypot(*d)).astype(f32) if (sx or sy) else (1.0, 0.0)
        pairs.append((A, B))
    dbg, _ = _run(pvb, oracle, H, W, dirs, pairs, thresh)
    assert (dbg["counts"].cpu().numpy()[0, :, 0] > 50).all()          # every keypoint has its designed winner


# ---- cone boundary, special norms, thresholds, several refit CTAs --------------------------------------------------
_NORMS = np.array([0.0, 1e-7, 1.1e-6, 1e4, 1e19, np.nan, np.inf, -np.inf])


def _adversarial_field(H, W, win, thresh, rng, frac_boundary=0.5, frac_special=0.08):
    """Directions at every pixel: on the winner's cone boundary at +-acos(t)*(1 + {0, +-1e-7}), towards it, random, or
    with one of the special norms."""
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    base = np.arctan2(float(win[1]) - ys, float(win[0]) - xs)
    th = np.arccos(np.clip(np.float64(f32(thresh)), -1, 1))
    side = rng.choice([-1.0, 1.0], (H, W))
    eps = rng.choice([1.0, 1 + 1e-7, 1 - 1e-7], (H, W))
    u = rng.uniform(size=(H, W))
    ang = np.where(u < frac_boundary, base + side * th * eps,
                   np.where(u < frac_boundary + 0.3, base, rng.uniform(0, 2 * np.pi, (H, W))))
    norm = np.where(rng.uniform(size=(H, W)) < frac_special, rng.choice(_NORMS, (H, W)), 1.0)
    with np.errstate(all="ignore"):
        v = np.stack([np.cos(ang), np.sin(ang)], -1) * norm[..., None]
    v[np.isinf(norm), 1] = 0.0                                       # (+-inf, 0)
    return v.astype(f32)


def _winners(H, W):
    """(target, pair, exact) per keypoint: winners at radius 0.5 from a pixel, inside the image, ~70 px and ~1e5 px
    outside it."""
    return [((f32(9.3), f32(6.4)), ((4, 2), (15, 9)), False),
            ((f32(W / 2 + 0.25), f32(H / 2 - 0.125)), ((3, 1), (W - 2, H - 3)), False),
            ((f32(W + 70.5), f32(H / 3)), ((W - 1, 0), (W - 5, H - 1)), False),
            ((f32(-1e5), f32(H / 2)), ((0, 0), (W - 1, H - 1)), False)]


@pytest.mark.parametrize("thresh", [-0.5, 0.0, 0.05, 0.5, 0.99, 0.999, 1.0])
def test_cone_boundary_special_norms_and_splits(pvb, oracle, thresh):
    """H x W = 48 x 128 = 6144 selected pixels = 3 refit CTAs per keypoint: boundary pixels, special norms and the sample
    pairs are spread over all of them."""
    H, W = 48, 128
    rng = np.random.default_rng(int(1000 * (thresh + 1)))
    wins = _winners(H, W)
    dirs = np.zeros((H, W, len(wins), 2), dtype=f32)
    pairs = []
    for k, (target, (A, B), exact) in enumerate(wins):
        vA, vB, h = _design_pair(oracle, A, B, target, exact)
        dirs[:, :, k] = _adversarial_field(H, W, h, thresh, rng)
        dirs[A[1], A[0], k], dirs[B[1], B[0], k] = vA, vB
        pairs.append((A, B))
    dbg, _ = _run(pvb, oracle, H, W, dirs, pairs, thresh)
    assert int(dbg["tn"][0]) == H * W
    if 0 < thresh < 1:
        assert (dbg["counts"].cpu().numpy()[0, :, 0] > 0).all()


def test_winner_at_the_prefilter_distance_limit(pvb, oracle):
    """Winner ~1e6 px from the image, placed so that |h-c|_1 of the image's pixels straddles the prefilter's 1e6 limit;
    the pixels sit on the cone boundary."""
    H, W = 16, 64
    rng = np.random.default_rng(77)
    A, B = (0, 0), (0, H - 1)
    cases = []
    for k, off in enumerate([1e6 + 8.0, 1e6 + W / 2, 1e6 + W - 8.0]):
        target = (f32(off), f32(0.0))                                 # |h-c|_1 = off - cx + cy
        vA, vB, h = _design_pair(oracle, A, B, target, exact=False)
        S = np.abs(float(h[0]) - np.arange(W))[None, :] + np.abs(float(h[1]) - np.arange(H))[:, None]
        assert S.min() < 1e6 < S.max(), (h, S.min(), S.max())
        cases.append((vA, vB, h))
    for thresh in (0.99, 0.5):
        dirs = np.zeros((H, W, len(cases), 2), dtype=f32)
        for k, (vA, vB, h) in enumerate(cases):
            dirs[:, :, k] = _adversarial_field(H, W, h, thresh, rng, frac_boundary=0.8, frac_special=0.0)
            dirs[A[1], A[0], k], dirs[B[1], B[0], k] = vA, vB
        _run(pvb, oracle, H, W, dirs, [(A, B)] * len(cases), thresh)


def test_no_votes_winner_at_origin(pvb, oracle):
    """Every count 0 (every pixel points away from the hypothesis): the winner is (0, 0) and the refit sums the pixels
    that happen to point at the origin."""
    H, W = 24, 40
    rng = np.random.default_rng(5)
    A, B = (10, 3), (30, 20)
    vA, vB, h = _design_pair(oracle, A, B, (f32(20.5), f32(12.25)), exact=False)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    away = np.arctan2(ys - float(h[1]), xs - float(h[0]))
    origin = np.arctan2(-ys, -xs)
    apart = np.abs(np.angle(-np.exp(1j * (origin - away)))) > 0.5     # the origin is > 0.5 rad off the direction to h
    ang = np.where((rng.uniform(size=(H, W)) < 0.5) & apart, origin, away)
    dirs = np.stack([np.cos(ang), np.sin(ang)], -1).astype(f32)[:, :, None]
    # the pair must not vote for its own intersection either: point both rays away (same lines, opposite directions)
    dirs[A[1], A[0], 0], dirs[B[1], B[0], 0] = -vA, -vB
    dbg, got = _run(pvb, oracle, H, W, dirs, [(A, B)], 0.99)
    assert (dbg["counts"].cpu().numpy() == 0).all()
    assert (dbg["win"].cpu().numpy() == 0).all()
    assert (dbg["normal_eq"].cpu().numpy()[0, 0, [0, 2]] > 100).all()   # the origin-pointing pixels were summed


def test_single_point_vote_tile_layer(pvb, oracle):
    """H x W = 6 x 256, rows 0-3 full plus pixel (3, 5): tn = 1025, so with hn = 300 (1024-pixel vote tiles) the last
    tile holds that pixel alone.  The winner is forced 1 ulp from it; the vote counts and the refit must both apply the
    reference's norm cut to it."""
    H, W = 6, 256
    mask = np.zeros((H, W), dtype=np.uint8)
    mask[:4] = 1
    mask[5, 3] = 1
    rng = np.random.default_rng(3)
    A, B = (3, 3), (10, 2)
    dirs = np.zeros((H, W, 3, 2), dtype=f32)
    targets = [(np.nextafter(f32(3), f32(4)), f32(5)), (f32(3), np.nextafter(f32(5), f32(4))), (f32(3), f32(5))]
    for k, target in enumerate(targets):
        dirs[:, :, k] = _towards(H, W, np.array(target, np.float64), rng)
        vA, vB, h = _design_pair(oracle, A, B, target)
        dirs[A[1], A[0], k], dirs[B[1], B[0], k] = vA, vB
    dirs[5, 3] = [(1, 0), (0, -1), (1, 0)]                           # pixel (3, 5) points at the winner
    dbg, _ = _run(pvb, oracle, H, W, dirs, [(A, B)] * 3, 0.99, hn=300, mask=mask)
    assert int(dbg["tn"][0]) == 1025
