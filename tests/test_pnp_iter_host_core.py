"""CPU: PVNet's default pose step (clean_pvnet_b200/csrc/pnp_iter_core.cuh, compiled as host code by
tests/pnp_iter_host_harness.cpp) against `cv2.solvePnP(..., flags=cv2.SOLVEPNP_ITERATIVE)` called exactly as
lib/utils/pvnet/pvnet_pose_utils.py:5-38 calls it.  OpenCV runs here, so the pin is against the real thing.

The bar: rvec and tvec within 1e-8 (max |difference| over max(1, max |OpenCV's value|)), and R of the returned 3x4 within
1e-8 of cv2.Rodrigues(rvec).  A problem counts as followable the way the Ceres pin decides it: OpenCV re-run on the image
points scaled by (1 + 1e-13) must not move by more than the bar; the others are counted, printed and excluded.

One more class escapes that test: once the loop has converged, a step changes |e| by a few ulps, so whether it counts as
raising |e| (and is retried with a 10x larger lambda) depends on the order in which the squares are summed.  OpenCV's
order is its own; the perturbation does not move that decision, but a different order can, and then the two solves stop
one step apart.  At most TIES_ALLOWED followable problems may land in (1e-8, 1e-7]; they are printed."""
import numpy as np
import pytest

from pnp_iter_cases import K_LINEMOD, STATUS, cases, host_core, opencv_pnp, rel_diff, _rotation

cv2 = pytest.importorskip("cv2")
BAR = 1e-8
MAX_UNFOLLOWABLE = 30          # of 3000: OpenCV's 20-iteration cap leaves a few problems mid-way on a flat valley
TIES_ALLOWED = 2               # of 3000: one occurs in this set, at 1.0005e-8


@pytest.fixture(scope="module")
def core():
    return host_core()


def test_matches_opencv_iterative(core):
    """3000 problems: pn in {6, 7, 9, 17, 33, 64}, noise 0 / 1 / 5 / 20 px, 0-2 vote outliers moved by 50-200 px, generic
    rotations and rotations near 0 and within 1e-7 of pi, depths 0.3-3 m, LINEMOD's and per-problem intrinsics."""
    cs = cases(3000)
    unfollowable = checked = 0
    worst = 0.0
    ties = []
    statuses = set()
    for pn in sorted({c[0].shape[0] for c in cs}):
        idx = [i for i, c in enumerate(cs) if c[0].shape[0] == pn]
        uv = np.stack([cs[i][0] for i in idx])
        X = np.stack([cs[i][1] for i in idx])
        K = np.stack([cs[i][2] for i in idx])
        pose, rt, info = core(uv, X, K)
        for j, i in enumerate(idx):
            want = opencv_pnp(X[j], uv[j], K[j])
            if rel_diff(want, opencv_pnp(X[j], uv[j] * (1 + 1e-13), K[j])) > BAR:
                unfollowable += 1
                continue
            checked += 1
            statuses.add(int(info[j, 1]))
            d = rel_diff(want, rt[j])
            bar = BAR
            if d > BAR:
                ties.append((i, d))
                bar = 10 * BAR
            else:
                worst = max(worst, d)
            assert d <= bar, (i, pn, d, info[j], want, rt[j])
            assert np.abs(pose[j, :, :3] - cv2.Rodrigues(want[:3])[0]).max() <= bar, i
            assert np.array_equal(pose[j, :, 3], rt[j, 3:])
    print(f"\n{checked} problems within {worst:.2e} of cv2 {cv2.__version__}; {unfollowable} excluded as not followable "
          f"(ceiling {MAX_UNFOLLOWABLE}); past 1e-8 on an accept-test tie: {ties}")
    assert checked + unfollowable == 3000 and unfollowable <= MAX_UNFOLLOWABLE and len(ties) <= TIES_ALLOWED
    assert statuses == {STATUS["ok"], STATUS["iteration_limit"]}      # on every followable problem


def test_shared_and_per_problem_intrinsics_and_model_agree(core):
    cs = [c for c in cases(400) if c[0].shape[0] == 9 and np.array_equal(c[2], K_LINEMOD)][:20]
    uv = np.stack([c[0] for c in cs])
    X = np.stack([c[1] for c in cs])
    per = core(uv, X, np.repeat(K_LINEMOD[None], len(cs), 0))
    shared_k = core(uv, X, K_LINEMOD)
    for a, b in zip(per, shared_k):
        assert np.array_equal(a, b)
    shared_m = core(uv[:1].repeat(3, 0), X[0], K_LINEMOD)
    assert np.array_equal(shared_m[1], per[1][:1].repeat(3, 0))


def test_rodrigues_matches_opencv(core):
    rng = np.random.default_rng(5)
    vecs = [rng.normal(size=3) * s for s in (1e-20, 1e-12, 1e-6, 0.3, 1.0, 3.0) for _ in range(20)]
    vecs += [np.zeros(3), np.array([np.pi, 0, 0]), np.array([0, 0, 1e-17])]
    for r in vecs:
        R, J = core.rodrigues(r)
        Rc, Jc = cv2.Rodrigues(r.reshape(3, 1))
        assert np.abs(R - Rc).max() <= 1e-15 and np.abs(J - Jc).max() <= 1e-14, r
    # matrix -> vector: generic, the identity, and within 1e-7 rad of pi (OpenCV's s < 1e-5 branch, which rebuilds the axis
    # from sqrt((R_ii + 1) / 2): a rounding error of R_ii becomes ~sqrt(DBL_EPSILON) there, in OpenCV as here)
    for k in range(200):
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        theta = [rng.uniform(0, np.pi), 0.0, np.pi - rng.uniform(0, 1e-7), np.pi][k % 4]
        R = _rotation(axis * theta)
        got, want = core.rotation_to_vector(R), cv2.Rodrigues(R)[0].ravel()
        assert np.abs(got - want).max() <= (1e-14 if k % 4 < 2 else 1e-7), (theta, got, want)


def _model(rng, pn, flatness):
    X = rng.uniform(-0.1, 0.1, (pn, 3))
    X[:, 2] *= flatness
    return X


def _project(X, K, rvec, t):
    return cv2.projectPoints(X, rvec, t, K, None)[0].reshape(-1, 2)


def _scatter_ratio(X):
    W = np.linalg.svd((X - X.mean(0)).T @ (X - X.mean(0)), compute_uv=False)
    return W[2] / W[1]


def test_too_few_points_and_the_planarity_threshold(core):
    """pn = 4 / 5 on a solid model: OpenCV raises (its DLT needs six points) and the core says too few points.  With pn = 5
    OpenCV's branch decision shows directly: below W[2]/W[1] = 1e-3 it solves through its homography start (the core
    reports a planar model), above it raises (too few points).  pn < 4 is too few for solvePnP itself."""
    rng = np.random.default_rng(11)
    rvec, t = np.array([0.3, -0.2, 0.1]), np.array([0.02, -0.01, 0.8])
    for pn, flat, want in ((4, 1.0, "too_few_points"), (5, 1.0, "too_few_points"), (5, 0.0195, None), (5, 0.098, None),
                           (9, 1e-3, "planar"), (3, 1.0, "too_few_points")):
        for _ in range(20):
            X = _model(rng, pn, flat)
            ratio = _scatter_ratio(X)
            if want is not None or (flat < 0.05 and 2e-4 < ratio < 6e-4) or (flat > 0.05 and 6e-3 < ratio < 1.2e-2):
                break
        uv = _project(X, K_LINEMOD, rvec, t)
        pose, rt, info = core(uv[None], X, K_LINEMOD)
        expect = want or ("planar" if ratio < 1e-3 else "too_few_points")
        assert info[0, 1] == STATUS[expect], (pn, ratio, info)
        assert np.isnan(pose).all() and np.isnan(rt).all()
        if expect == "planar":
            assert np.abs(opencv_pnp(X, uv, K_LINEMOD) - np.r_[rvec, t]).max() < 1e-6      # OpenCV solves it
        else:
            with pytest.raises(cv2.error):
                opencv_pnp(X, uv, K_LINEMOD)


def test_nan_points_are_degenerate(core):
    uv, X, K = cases(1, seed0=77)[0]
    for where in ((0, 0), (3, 1)):
        u = uv.copy()
        u[where] = np.nan
        pose, rt, info = core(u[None], X, K)
        assert info[0, 1] == STATUS["degenerate"] and np.isnan(pose).all()
        with pytest.raises(cv2.error):
            opencv_pnp(X, u, K)
    Xn = X.copy()
    Xn[2, 0] = np.inf
    assert core(uv[None], Xn, K)[2][0, 1] == STATUS["degenerate"]


def test_skipped_image_is_degenerate_and_fails_every_flag_either_way(core):
    """The voting layer returns kpt = 0 for an image it skipped.  OpenCV then returns a finite, meaningless pose; the core
    reports degenerate with a NaN pose.  Both fail all three pose flags of the restated evaluator
    (lib/evaluators/linemod/pvnet.py:59-94: 2-D projection < 5 px, ADD < 0.1 diameter, 5 cm 5 degrees)."""
    rng = np.random.default_rng(2)
    model = rng.normal(size=(500, 3)) * [0.05, 0.03, 0.04]
    kpt3d = np.concatenate([model[:8], model.mean(0, keepdims=True)])
    diameter = float(np.max(np.linalg.norm(model[:, None] - model[None, ::5], axis=-1)))
    uv = np.zeros((9, 2))
    pose, rt, info = core(uv[None], kpt3d, K_LINEMOD)
    assert info[0, 1] == STATUS["degenerate"] and np.isnan(pose).all() and np.isnan(rt).all()
    cvrt = opencv_pnp(kpt3d, uv, K_LINEMOD)
    assert np.isfinite(cvrt).all()
    cv_pose = np.concatenate([cv2.Rodrigues(cvrt[:3])[0], cvrt[3:, None]], 1)

    def flags(p, gt):
        def proj(q):
            c = (model @ q[:, :3].T + q[:, 3]) @ K_LINEMOD.T
            with np.errstate(divide="ignore", invalid="ignore"):
                return c[:, :2] / c[:, 2:]
        with np.errstate(invalid="ignore"):
            p2d = np.mean(np.linalg.norm(proj(p) - proj(gt), axis=-1)) < 5
            add = np.mean(np.linalg.norm((model @ p[:, :3].T + p[:, 3]) - (model @ gt[:, :3].T + gt[:, 3]), axis=-1))
            tr = np.trace(p[:, :3] @ gt[:, :3].T)
        tr = tr if tr <= 3 else 3
        tr = tr if tr >= -1 else -1
        cmd5 = np.linalg.norm(p[:, 3] - gt[:, 3]) * 100 < 5 and np.rad2deg(np.arccos((tr - 1.0) / 2.0)) < 5
        return bool(p2d), bool(add < diameter * 0.1), bool(cmd5)

    for k in range(20):
        gt = np.concatenate([_rotation(rng.normal(size=3)), [[rng.uniform(-0.1, 0.1)], [rng.uniform(-0.1, 0.1)],
                                                            [rng.uniform(0.5, 1.2)]]], 1)
        assert flags(cv_pose, gt) == flags(pose[0], gt) == (False, False, False)
