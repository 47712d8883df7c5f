"""Shared helpers for the GPU parity tests."""
import numpy as np
import torch


def field_case(tn=2000, vn=3, hn=128, seed=0, noise_deg=3.0, outliers=0.2, extent=(640, 480)):
    """Reference-layout inputs: direct [tn,vn,2], coords [tn,2] (integer pixels), idxs [hn,vn,2]."""
    rng = np.random.default_rng(seed)
    W, H = extent
    coords = np.stack([rng.integers(0, W, tn), rng.integers(0, H, tn)], axis=1).astype(np.float32)
    kp = np.stack([rng.uniform(0.1 * W, 0.9 * W, vn), rng.uniform(0.1 * H, 0.9 * H, vn)], axis=1)
    kp[-1, 0] = 1.3 * W
    ang = np.arctan2(kp[None, :, 1] - coords[:, None, 1], kp[None, :, 0] - coords[:, None, 0])
    ang = ang + rng.normal(0, np.radians(noise_deg), size=ang.shape)
    out = rng.uniform(size=ang.shape) < outliers
    ang = np.where(out, rng.uniform(0, 2 * np.pi, size=ang.shape), ang)
    direct = np.stack([np.cos(ang), np.sin(ang)], axis=-1).astype(np.float32)
    idxs = rng.integers(0, tn, size=(hn, vn, 2)).astype(np.int32)
    idxs[0, :, 1] = idxs[0, :, 0]                       # t0 == t1 -> degenerate
    return direct, coords, idxs, kp.astype(np.float32)


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def bits_equal(a, b):
    a = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    b = np.ascontiguousarray(b, dtype=np.float32).view(np.uint32)
    return np.array_equal(a, b)


def normal_eq_of_inliers(dirs, xy, inl):
    """The refit's normal equations over the pixels flagged in `inl` (ransac_voting_gpu.py:177-191), in float64:
    normal n = (v_y, -v_x), b = n.c; returns ((a00, a01, a11, b0, b1), sum over the same terms of |term|, inlier count).
    dirs [tn,2] float32, xy [tn,2] float32, inl [tn] bool."""
    v = np.asarray(dirs, dtype=np.float64)[inl]
    c = np.asarray(xy, dtype=np.float64)[inl]
    nx, ny = v[:, 1], -v[:, 0]
    bb = nx * c[:, 0] + ny * c[:, 1]
    terms = np.stack([nx * nx, nx * ny, ny * ny, nx * bb, ny * bb])
    return terms.sum(axis=1), np.abs(terms).sum(axis=1), int(inl.sum())


def reference_normal_eq(dbg, thresh, inliers_of):
    """What the refit must sum, per (image, keypoint): the reference predicate applied to the winner
    (voting_for_hypothesis with hn = 1, hyp = win) over the image's selected pixels.  `inliers_of(direct [tn,K,2],
    coords [tn,2], hyp [1,K,2], thresh)` returns the uint8 inlier bytes [1,K,tn].  Returns float64 [B,K,5] sums, the
    matching |term| sums and int [B,K] inlier counts; skipped images give zeros."""
    tn = dbg["tn"].cpu().numpy()
    state = dbg["state"].cpu().numpy()
    B, K = dbg["win"].shape[:2]
    eq, scale, cnt = np.zeros((B, K, 5)), np.zeros((B, K, 5)), np.zeros((B, K), dtype=np.int64)
    for b in range(B):
        n = int(tn[b])
        if state[b] != 0 or n <= 0:
            continue
        xy = dbg["xy"][b, :n].cpu().numpy()
        direct = dbg["dirs"][b, :, :n].permute(1, 0, 2).contiguous().cpu().numpy()      # [tn,K,2]
        hyp = dbg["win"][b][None].cpu().numpy()                                         # [1,K,2]
        inl = inliers_of(direct, xy, hyp, thresh)
        for k in range(K):
            eq[b, k], scale[b, k], cnt[b, k] = normal_eq_of_inliers(direct[:, k], xy, inl[0, k] != 0)
    return eq, scale, cnt


def oracle_inliers(oracle):
    def inliers_of(direct, coords, hyp, thresh):
        out = np.zeros((1, direct.shape[1], direct.shape[0]), dtype=np.uint8)
        with np.errstate(all="ignore"):
            oracle.voting_for_hypothesis(direct, coords, hyp, out, thresh)
        return out
    return inliers_of


def twin_inliers(pvb):
    """The same bytes from the repo's CUDA twin of the reference's voting_for_hypothesis (pinned to the reference's
    stored output in test_gpu_reference_parity.py): for images too large for the CPU oracle."""
    def inliers_of(direct, coords, hyp, thresh):
        d, c, h = cuda(direct, coords, hyp)
        out = torch.zeros((1, direct.shape[1], direct.shape[0]), dtype=torch.uint8, device="cuda")
        pvb.ransac_voting.voting_for_hypothesis(d, c, h, out, thresh)
        return out.cpu().numpy()
    return inliers_of


NEQ_RTOL = 1e-12     # the only difference left is the order of the float64 sums


def check_normal_eq(dbg, thresh, inliers_of):
    """The refit's normal equations (debug `normal_eq`) equal the sums over the reference predicate's inliers of the
    winner up to float64 summation order, and the inlier count equals the winner's vote count.  One pixel too many or too
    few changes a00 + a11 by |v|^2, far outside the bar.  Returns the reference inlier counts [B,K]."""
    got = dbg["normal_eq"].cpu().numpy()
    want, scale, cnt = reference_normal_eq(dbg, thresh, inliers_of)
    assert got.shape == want.shape and got.dtype == np.float64
    err = np.abs(got - want)
    bad = ~(err <= NEQ_RTOL * scale)
    assert not bad.any(), f"normal_eq mismatch at {np.argwhere(bad)[:5].tolist()}: got {got[bad][:5]}, want {want[bad][:5]}"
    counts = dbg["counts"].cpu().numpy()
    best = counts.max(axis=2) if counts.shape[2] else np.zeros(cnt.shape, dtype=counts.dtype)
    voted = best > 0
    assert np.array_equal(cnt[voted], best[voted])
    return cnt


def pnp_case(seed, pn=9, noise=1.0, pert=(0.05, 0.02)):
    """One synthetic uncertainty-PnP problem in the LINEMOD geometry (model points within +-10 cm, object 0.6-1.2 m away,
    LINEMOD intrinsics): (pts2d [pn,2], pts3d [pn,3], wgt2d [pn,3], K [3,3], init_rt [6], true_rt [6]), float64.
    Weights are inv(sqrtm(cov)) of random SPD covariances, i.e. what pvb_uncertainty_weights produces."""
    rng = np.random.default_rng(seed)
    pts3d = rng.uniform(-0.1, 0.1, (pn, 3))
    aa = rng.normal(size=3)
    aa *= rng.uniform(0.2, 2.5) / np.linalg.norm(aa)
    t = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(0.6, 1.2)])
    K = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1.0]])
    theta = np.linalg.norm(aa)
    w = aa / theta
    Wx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    R = np.eye(3) + np.sin(theta) * Wx + (1 - np.cos(theta)) * (Wx @ Wx)
    cam = pts3d @ R.T + t
    uv = np.stack([K[0, 0] * cam[:, 0] / cam[:, 2] + K[0, 2], K[1, 1] * cam[:, 1] / cam[:, 2] + K[1, 2]], 1)
    uv = uv + rng.normal(size=uv.shape) * noise
    wgt = np.empty((pn, 3))
    for i in range(pn):
        A = rng.normal(size=(2, 2))
        C = A @ A.T * rng.uniform(0.5, 4) + 0.1 * np.eye(2)
        lam, V = np.linalg.eigh(C)
        Wi = V @ np.diag(lam ** -0.5) @ V.T
        wgt[i] = [Wi[0, 0], Wi[0, 1], Wi[1, 1]]
    true_rt = np.concatenate([aa, t])
    init = true_rt + np.concatenate([rng.normal(size=3) * pert[0], rng.normal(size=3) * pert[1]])
    return uv, pts3d, wgt, K, init, true_rt


def restated_covariance(dbg, mean):
    """float64 restatement of covariance_kernel (ransac_voting_gpu.py:243-244, 254-269) from the distribution op's
    debug `hyp` [B,K,hn,2] and `counts` [B,K,hn]: ratio = fp32(count) / fp32(tn) (skipped images: hyp 0, ratio 1),
    th = fp32(max - 0.1f), w = 0 where w < th, d = fp32(hyp - mean), S = sum w*d*d^T in float64,
    den = fp32(fp32(sum w) + 1e-3f).  Returns (S / den as float64 [B,K,2,2], the matching sums of |term| / den)."""
    hyp = dbg["hyp"].cpu().numpy()
    counts = dbg["counts"].cpu().numpy()
    tn = dbg["tn"].cpu().numpy()
    skipped = (dbg["state"].cpu().numpy() != 0)[:, None, None]
    mean = np.asarray(mean.cpu() if isinstance(mean, torch.Tensor) else mean, dtype=np.float32)
    with np.errstate(all="ignore"):
        ratio = np.where(skipped, np.float32(1), counts.astype(np.float32) / tn.astype(np.float32)[:, None, None])
        hyp = np.where(skipped[..., None], np.float32(0), hyp)
        th = (ratio.max(axis=2) - np.float32(0.1)).astype(np.float32)
        w = np.where(ratio < th[..., None], np.float32(0), ratio).astype(np.float64)
        d = (hyp - mean[:, :, None, :]).astype(np.float64)               # fp32 difference, then widened
        t00, t01, t11 = d[..., 0] * (d[..., 0] * w), d[..., 0] * (d[..., 1] * w), d[..., 1] * (d[..., 1] * w)
        den = (np.float32(w.sum(axis=2)) + np.float32(1e-3)).astype(np.float64)
        S = np.stack([t00.sum(2), t01.sum(2), t01.sum(2), t11.sum(2)], -1).reshape(hyp.shape[:2] + (2, 2))
        A = np.stack([np.abs(t00).sum(2), np.abs(t01).sum(2), np.abs(t01).sum(2), np.abs(t11).sum(2)], -1)
        return S / den[..., None, None], A.reshape(S.shape) / den[..., None, None]


def check_covariance(cov, dbg, mean):
    """The op's covariance against restated_covariance: every entry within 1 fp32 ulp of the float64 value, plus
    1e-12 * sum|terms| / den (float64 summation order, matters only for off-diagonals that cancel to ~0); NaN exactly
    where the restatement is NaN; the two off-diagonals bit-equal.  Returns the restated float64 covariance."""
    got = cov.cpu().numpy().astype(np.float64)
    want, scale = restated_covariance(dbg, mean)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), np.argwhere(np.isnan(got) != nan)[:5]
    bar = np.spacing(np.abs(want[~nan]).astype(np.float32)).astype(np.float64) + 1e-12 * scale[~nan]
    err = np.abs(got[~nan] - want[~nan])
    assert (err <= bar).all(), f"cov off by {np.max(err / bar):.2f}x the bar; got {got[~nan][err > bar][:4]}, want {want[~nan][err > bar][:4]}"
    c = cov.cpu().numpy()
    assert bits_equal(c[..., 0, 1], c[..., 1, 0])
    return want
