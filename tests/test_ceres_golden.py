"""CPU: the pin of SURVEY 8f row 3 against the reference itself.

tests/golden/ceres_pnp.npz holds 284 problems solved by REAL Ceres 2.0 (the reference's prebuilt libceres.so.2.0.0 + its
unmodified src/uncertainty_pnp.cpp, tests/golden/make_golden_ceres.py).  Checked here, without a GPU:
  * oracle/pnp_oracle.py (the numpy restatement) follows Ceres: same stop reason, same number of iterations, same cost after
    every iteration, same pose (1e-9) -- including descents with up to 20 rejected steps and the 50-iteration cap;
  * the arithmetic core of the CUDA kernel (csrc/pnp_core.cuh compiled as host code) does the same.
tests/golden/ceres_pnp_fp32.npz (228 problems with the fused tail's fp32 inputs, tests/golden/make_golden_ceres_fp32.py) is
held to the same bar from three starts each, below.
Iteration bookkeeping: Ceres appends an IterationSummary when an iteration is finalised; an iteration that ends the solve by
the parameter- or function-tolerance test returns before that (trust_region_minimizer.cc), so for those reasons
#summaries == iterations started (summary 0 is the initial evaluation), otherwise #summaries - 1."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "ceres_pnp.npz"))
N = len(G["pn"])


def problem(i):
    pn = int(G["pn"][i])
    return G["pts2d"][i, :pn], G["pts3d"][i, :pn], G["wgt2d"][i, :pn], G["K"][i], G["init_rt"][i]


def expected_iterations(i):
    return int(G["iteration_summaries"][i]) - (0 if G["reason"][i] in (2, 3) else 1)


def followable(i):
    return bool(G["stable"][i]) and G["kind"][i] != "optimum"


def test_fixture_shape():
    assert N == 284 and (G["linear_solver_type_used"] == 3).all()           # DENSE_SCHUR, as uncertainty_pnp.cpp:84 asks
    assert sum(followable(i) for i in range(N)) >= 230
    assert int(G["unsuccessful"][[followable(i) for i in range(N)]].max()) >= 15   # rejected steps are covered
    assert (G["reason"][[followable(i) for i in range(N)]] == 5).sum() >= 10       # and so is the iteration cap
    assert np.array_equal(G["result_rt"], G["entry_rt"], equal_nan=True)   # probe == the reference's own C entry


def test_oracle_follows_ceres():
    import pnp_oracle as po
    worst = 0.0
    for i in range(N):
        with np.errstate(all="ignore"):
            x, info = po.uncertainty_pnp(*problem(i), return_info=True)
        if not followable(i):
            if G["kind"][i] == "optimum":                                  # costs ~1e-20: only the pose is meaningful
                assert np.abs(x - G["result_rt"][i]).max() < 1e-8, i
            continue
        assert info["termination"] == G["reason"][i], i
        assert info["iterations"] == expected_iterations(i), i
        d = np.abs(x - G["result_rt"][i]).max()
        worst = max(worst, d)
        assert d < 1e-9, (i, d)
        assert abs(info["cost"] - G["final_cost"][i]) <= 1e-9 * G["final_cost"][i], i
    assert worst < 1e-9


@pytest.fixture(scope="module")
def host_core():
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libpnp_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-ffp-contract=off", "-x", "c++",
                           os.path.join(ROOT, "tests", "pnp_host_harness.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    DP = ctypes.POINTER(ctypes.c_double)

    def solve(uv, p3, W, K, init):
        a = [np.ascontiguousarray(v, np.float64) for v in (uv, p3, W, K, init)]
        res, info = np.empty(6), (ctypes.c_int * 2)()
        lib.pnp_host_solve(*[v.ctypes.data_as(DP) for v in a], res.ctypes.data_as(DP), info, ctypes.c_int(len(uv)),
                           ctypes.c_int(50), ctypes.c_double(1e-6), ctypes.c_double(1e-10), ctypes.c_double(1e-8))
        return res, info[0], info[1]
    return solve


def test_cuda_core_follows_ceres(host_core):
    """csrc/pnp_core.cuh (the code the kernel runs, compiled for the host) against real Ceres."""
    for i in range(N):
        if not followable(i):
            continue
        x, it, code = host_core(*problem(i))
        assert (it, code) == (expected_iterations(i), G["reason"][i]), i
        assert np.abs(x - G["result_rt"][i]).max() < 1e-9, i


# ---------------------------------------------------------------------------------------------------------------------
# tests/golden/ceres_pnp_fp32.npz: the inputs the fused tail sees (fp32 keypoints, fp32 covariances and the fp32 weights
# cov_to_weights makes of them, float64 model and camera), at the production point counts 9 and 17, across the warp's
# one-point-per-lane boundary up to the fused kernel's 64, with zero-weight keypoints, skipped images and pn = 3 / 4; each
# problem solved by Ceres from a perturbed true pose (no prefix) and from OpenCV's P3P pose on the default-kind (`p3p_`)
# and the stable (`p3ps_`) argsort top four (tests/golden/make_golden_ceres_fp32.py).  The GPU side is
# tests/test_gpu_pnp_tail.py; this file checks that the fixture can be followed at all before a kernel is held to it.
F = np.load(os.path.join(ROOT, "tests", "golden", "ceres_pnp_fp32.npz"))
NF = len(F["pn"])
START = ("", "p3p_", "p3ps_")


def f_problem(i, start=""):
    pn = int(F["pn"][i])
    init = F["init_rt"][i] if start == "" else F[start[:-1] + "_rt"][i]
    return (F["kpt2d"][i, :pn].astype(np.float64), F["pts3d"][i, :pn], F["wgt2d"][i, :pn].astype(np.float64), F["K"][i], init)


def f_expected(i, start=""):
    """(iterations, stop reason) Ceres reports for fixture problem i from the given start."""
    reason = int(F[start + "reason"][i])
    return int(F[start + "iteration_summaries"][i]) - (0 if reason in (2, 3) else 1), reason


def f_followable(i, start=""):
    return bool(F[start + "stable"][i]) and int(F["pn"][i]) >= (1 if start == "" else 4)


def test_fp32_fixture_shape():
    from util import cov_to_weights_f32
    assert NF == 228 and F["kpt2d"].dtype == np.float32 and F["cov"].dtype == np.float32 and F["wgt2d"].dtype == np.float32
    hist = {int(p): int(c) for p, c in zip(*np.unique(F["pn"], return_counts=True))}
    assert hist == {3: 8, 4: 8, 9: 82, 17: 82, 31: 8, 32: 8, 33: 8, 48: 8, 63: 8, 64: 8}
    kinds = {str(k): int(c) for k, c in zip(*np.unique(F["kind"], return_counts=True))}
    assert kinds == {"prod9": 64, "prod17": 64, "wide": 48, "zeros": 32, "skipped": 4, "small": 16}
    assert [sum(f_followable(i, s) for i in range(NF)) for s in START] == [228, 215, 215]
    # the weights are cov_to_weights' rule on the stored covariances, bit for bit, and nothing beyond pn is set
    for i in range(NF):
        pn = int(F["pn"][i])
        assert np.array_equal(F["wgt2d"][i, :pn], cov_to_weights_f32(F["cov"][i, :pn])), i
        assert not F["kpt2d"][i, pn:].any() and not F["wgt2d"][i, pn:].any() and not F["pts3d"][i, pn:].any()
    # the sets are what they claim to be: one model and camera per shared set, zero keys, negative keys, skipped images
    for kind in ("prod9", "prod17"):
        m = np.nonzero(F["kind"] == kind)[0]
        assert F["shared"][m].all() and (F["pts3d"][m] == F["pts3d"][m[0]]).all() and (F["K"][m] == F["K"][m[0]]).all()
    w = F["wgt2d"].astype(np.float64)
    key = w[..., 0] + w[..., 1]
    live = np.arange(64)[None] < F["pn"][:, None]
    z = F["kind"] == "zeros"
    assert ((key[z] == 0) & live[z]).any(1).all() and ((key[z] < 0) & live[z]).sum() >= 10
    assert (((key > 0) & live).sum(1)[z] < 4).sum() >= 8                    # fewer than four positive keys
    assert np.isnan(F["cov"][z]).any() and not np.isnan(F["wgt2d"]).any()
    s = F["kind"] == "skipped"
    assert not F["kpt2d"][s].any() and not F["cov"][s].any() and not F["wgt2d"][s].any()
    assert str(F["numpy_version"]) and str(F["opencv_version"])


def test_fp32_fixture_weights_are_inv_sqrtm():
    """The stored fp32 weights against scipy's inv(sqrtm(cov)) -- what lib/evaluators/linemod/pvnet.py:118-130 computes --
    within 2 fp32 ulp (the bar of test_uncertainty_pnp_weights_sweep), and zero exactly where the reference zeroes them."""
    import scipy.linalg
    for i in range(NF):
        for j in range(int(F["pn"][i])):
            c, w = F["cov"][i, j], F["wgt2d"][i, j]
            if c[0, 0] < 1e-6 or np.isnan(c).any():
                assert not w.any(), (i, j)
                continue
            m = np.linalg.inv(scipy.linalg.sqrtm(c.astype(np.float64)))
            want = np.array([m[0, 0], m[0, 1], m[1, 1]])
            bar = 2 * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + 1e-12 * np.abs(want).max()
            assert (np.abs(w - want) <= bar).all(), (i, j, w, want)


@pytest.mark.parametrize("start", START)
def test_oracle_follows_ceres_fp32(start):
    import pnp_oracle as po
    for i in range(NF):
        if not f_followable(i, start):
            continue
        with np.errstate(all="ignore"):
            x, info = po.uncertainty_pnp(*f_problem(i, start), return_info=True)
        assert (info["iterations"], info["termination"]) == f_expected(i, start), (start, i)
        assert np.abs(x - F[start + "result_rt"][i]).max() < 1e-9, (start, i)


@pytest.mark.parametrize("start", START)
def test_cuda_core_follows_ceres_fp32(host_core, start):
    for i in range(NF):
        if not f_followable(i, start):
            continue
        x, it, code = host_core(*f_problem(i, start))
        assert (it, code) == f_expected(i, start), (start, i)
        assert np.abs(x - F[start + "result_rt"][i]).max() < 1e-9, (start, i)


def test_unfollowable_starts_are_the_ones_without_a_p3p_pose():
    """Every problem Ceres cannot be followed on from a P3P start is one where OpenCV returned no finite pose (a skipped
    image, a degenerate triple) or pn < 4; from the perturbed truth every problem is followable."""
    for i in range(NF):
        for s in ("p3p_", "p3ps_"):
            if not f_followable(i, s):
                assert int(F["pn"][i]) < 4 or not np.isfinite(F[s[:-1] + "_rt"][i]).all(), (s, i)

