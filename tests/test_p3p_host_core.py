"""CPU: the closed-form initial pose of the uncertainty PnP (clean_pvnet_b200/csrc/p3p_core.cuh, compiled as host code by
tests/p3p_host_harness.cpp) against the reference's own initialiser, `cv2.solvePnP(..., flags=cv2.SOLVEPNP_P3P)` called exactly
as un_pnp_utils.py:25-31 calls it.  OpenCV runs here, so this pin is against the real thing, not a restatement."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from util import pnp_case

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DP = ctypes.POINTER(ctypes.c_double)


@pytest.fixture(scope="module")
def p3p():
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libp3p_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "p3p_host_harness.cpp"), "-o", so])
    lib = ctypes.CDLL(so)

    def solve(X, x2, K):
        X, x2, K = [np.ascontiguousarray(a, np.float64) for a in (X, x2, K)]
        rt = np.full(6, np.nan)
        n = lib.p3p_host_solve4(X.ctypes.data_as(DP), x2.ctypes.data_as(DP), K.ctypes.data_as(DP), rt.ctypes.data_as(DP))
        return n, rt

    def quartic(k):
        k = np.ascontiguousarray(k, np.float64)
        out = np.zeros(4)
        n = lib.p3p_host_quartic(k.ctypes.data_as(DP), out.ctypes.data_as(DP))
        return np.sort(out[:n])

    def select4(w):
        w = np.ascontiguousarray(w, np.float64)
        idx = (ctypes.c_int * 4)()
        lib.p3p_host_select4(w.ctypes.data_as(DP), ctypes.c_int(len(w)), idx)
        return list(idx)

    solve.quartic = quartic
    solve.select4 = select4
    return solve


def _rodrigues(aa):
    return cv2.Rodrigues(np.asarray(aa, np.float64).reshape(3, 1))[0]


def _reproject(rt, X, K):
    c = X @ _rodrigues(rt[:3]).T + rt[3:]
    return np.stack([K[0, 0] * c[:, 0] / c[:, 2] + K[0, 2], K[1, 1] * c[:, 1] / c[:, 2] + K[1, 2]], 1)


def test_quartic_real_roots(p3p):
    rng = np.random.default_rng(0)
    for _ in range(1500):
        nreal = int(rng.choice([0, 2, 4]))
        roots = list(rng.normal(size=nreal) * rng.choice([0.1, 1, 10]))
        poly = np.poly1d([1.0])
        for x in roots:
            poly *= np.poly1d([1, -x])
        for _ in range((4 - nreal) // 2):
            re, im = rng.normal(), abs(rng.normal()) + 0.1
            poly *= np.poly1d([1, -2 * re, re * re + im * im])
        got = p3p.quartic((poly.coeffs * rng.uniform(0.5, 3))[::-1])
        want = np.sort(np.array(roots))
        assert len(got) == len(want)
        if nreal:
            assert np.abs(got - want).max() <= 1e-6 * (1 + np.abs(want).max())
    assert len(p3p.quartic([1.0, 0.0, -2.0, 0.0, 1.0])) == 4          # (x^2-1)^2: double roots, biquadratic branch
    assert len(p3p.quartic([1.0, 2.0, 3.0, 4.0, 0.0])) == 0          # leading coefficient 0: not a quartic


def test_selected_pose_matches_opencv_p3p(p3p):
    """3000 LINEMOD-like problems, noise 0 / 1 / 5 px: same pose as cv2.solvePnP(P3P) to 1e-6 whenever OpenCV's own ranking of the
    candidate poses is not a tie; the three P3P points reproject exactly (1e-8 px)."""
    ties = nan_cv = 0
    for s in range(3000):
        uv, p3, W, K, _, _ = pnp_case(2000 + s, pn=9, noise=[0.0, 1.0, 5.0][s % 3])
        idx = np.argsort(W[:, 0] + W[:, 1])[-4:]                      # un_pnp_utils.py:25
        X, x2 = p3[idx], uv[idx]
        n, rt = p3p(X, x2, K)
        ok, rvec, tvec = cv2.solvePnP(np.expand_dims(X, 0), np.expand_dims(x2, 0), K, np.zeros((8, 1)), None, None, False,
                                      flags=cv2.SOLVEPNP_P3P)
        if not (np.isfinite(rvec).all() and np.isfinite(tvec).all()):   # OpenCV returns NaN on a few degenerate triples
            nan_cv += 1
            assert n == 0 and np.isnan(rt).all()                       # ours reports "no admissible solution", pose untouched
            continue
        assert n >= 1
        assert np.abs(_reproject(rt, X[:3], K) - x2[:3]).max() < 1e-8
        d = max(np.abs(_rodrigues(rt[:3]) - _rodrigues(rvec)).max(), np.abs(rt[3:] - tvec.ravel()).max())
        if d > 1e-6:
            # a different root: only legitimate if the fourth point cannot tell the candidates apart (errors within 0.1 %)
            e_ours = np.linalg.norm(_reproject(rt, X[3:], K) - x2[3:])
            e_cv = np.linalg.norm(_reproject(np.concatenate([rvec.ravel(), tvec.ravel()]), X[3:], K) - x2[3:])
            assert abs(e_ours - e_cv) <= 1e-3 * e_cv and e_ours <= e_cv * (1 + 1e-9), s
            ties += 1
    assert ties <= 3 and nan_cv <= 6


def test_exact_data_recovers_the_true_pose(p3p):
    for s in range(50):
        uv, p3, W, K, _, true_rt = pnp_case(6000 + s, pn=9, noise=0.0)
        idx = np.argsort(W[:, 0] + W[:, 1])[-4:]
        n, rt = p3p(p3[idx], uv[idx], K)
        assert n >= 1
        assert np.abs(_rodrigues(rt[:3]) - _rodrigues(true_rt[:3])).max() < 1e-7 and np.abs(rt[3:] - true_rt[3:]).max() < 1e-7


def test_degenerate_triples_report_no_solution(p3p):
    uv, p3, W, K, _, _ = pnp_case(7000, pn=9, noise=0.0)
    X, x2 = p3[:4].copy(), uv[:4].copy()
    X[1] = X[0]                                                        # two identical model points
    n, rt = p3p(X, x2, K)
    assert n == 0 and np.isnan(rt).all()
    X = p3[:4].copy()
    X[2] = X[0] + 2.0 * (X[1] - X[0])                                  # collinear model points
    n, rt = p3p(X, x2, K)
    assert n == 0 and np.isnan(rt).all()
    for pt in ([0.0, 0.0], uv[0]):                                     # coincident image points (a skipped image: all 0)
        n, rt = p3p(p3[:4], np.tile(pt, (4, 1)), K)
        assert n == 0 and np.isnan(rt).all()


def test_selection_of_the_four_best_weighted_points(p3p):
    """`np.argsort(weights_2d[:, 0] + weights_2d[:, 1])[-4:]` (un_pnp_utils.py:25) with a stable sort, ties and NaNs included."""
    rng = np.random.default_rng(3)
    for trial in range(300):
        pn = int(rng.integers(4, 18))
        w = rng.normal(size=(pn, 3))
        if trial % 3 == 0:
            w[:, :2] = rng.integers(0, 3, size=(pn, 2))            # many ties
        if trial % 7 == 0:
            w[rng.integers(0, pn), 0] = np.nan
        want = list(np.argsort(w[:, 0] + w[:, 1], kind="stable")[-4:])
        assert p3p.select4(w) == want, (trial, w)


def test_tied_keys_take_the_stable_tail(p3p):
    """The tie rule, pinned: among equal keys the larger index ranks higher (the tail of a stable ascending argsort).  The
    reference calls np.argsort with numpy's default kind, whose order among ties depends on the sort implementation numpy
    was built with and dispatches to (with numpy 2.3 on an AVX-512 host it picks [13 15 16 3] here); this project keeps
    the stable tail, so the choice does not depend on the machine (DESIGN.md section 8 row 3)."""
    w = np.zeros((17, 3))
    w[3, 0] = 1.0
    assert p3p.select4(w) == [14, 15, 16, 3] == list(np.argsort(w[:, 0] + w[:, 1], kind="stable")[-4:])
    w = np.zeros((9, 3))
    w[2, 1] = 2.0
    w[[0, 4], 0] = -0.5                                               # negative keys rank below the zero-weight keypoints
    assert p3p.select4(w) == [6, 7, 8, 2]
    assert p3p.select4(np.zeros((9, 3))) == [5, 6, 7, 8]              # a skipped image: the last four keypoints


def _fp32_fixture():
    return np.load(os.path.join(ROOT, "tests", "golden", "ceres_pnp_fp32.npz"))


def test_fp32_fixture_p3p_matches_stored_opencv(p3p):
    """tests/golden/ceres_pnp_fp32.npz stores OpenCV's P3P pose on the stable top four (`p3ps_rt`) of every problem with
    pn >= 4: p3p_select4 picks those four, and p3p_solve4 gives OpenCV's pose to 1e-6 unless the fourth point cannot tell
    the candidates apart (the allowance of test_selected_pose_matches_opencv_p3p); where OpenCV has no finite pose (the
    skipped images: four coincident image points) it reports no solution."""
    F = _fp32_fixture()
    ties = checked = 0
    for i in range(len(F["pn"])):
        pn = int(F["pn"][i])
        if pn < 4:
            continue
        w = F["wgt2d"][i, :pn].astype(np.float64)
        idx = p3p.select4(w)
        assert idx == F["idx_stable"][i].tolist(), i
        uv, X, K = F["kpt2d"][i, :pn].astype(np.float64)[idx], F["pts3d"][i, :pn][idx], F["K"][i]
        n, rt = p3p(X, uv, K)
        want = F["p3ps_rt"][i]
        if not np.isfinite(want).all():
            assert n == 0 and np.isnan(rt).all(), i
            continue
        checked += 1
        assert n >= 1, i
        d = max(np.abs(_rodrigues(rt[:3]) - _rodrigues(want[:3])).max(), np.abs(rt[3:] - want[3:]).max())
        if d > 1e-6:
            e_ours = np.linalg.norm(_reproject(rt, X[3:], K) - uv[3:])
            e_cv = np.linalg.norm(_reproject(want, X[3:], K) - uv[3:])
            assert abs(e_ours - e_cv) <= 1e-3 * e_cv and e_ours <= e_cv * (1 + 1e-9), i
            ties += 1
    assert checked >= 200 and ties <= 2
    # where the two sort kinds picked the same four, the reference's own start is the stored stable one
    same = (F["idx_default"] == F["idx_stable"]).all(1)
    assert np.array_equal(F["p3p_rt"][same], F["p3ps_rt"][same], equal_nan=True)
    assert (~same).sum() >= 4 and (F["kind"][~same] == "zeros").all()              # ties only where keys are zero
