"""GPU: the batched uncertainty-PnP kernel (pvb_uncertainty_pnp, csrc/pnp.cu) against the oracle (oracle/pnp_oracle.py).

Tolerances (float64 throughout): where kernel and oracle take the same number of iterations and stop for the same reason the
poses agree to 1e-9 (the warp's butterfly sum and the oracle's BLAS sum differ in the last bits only); a last-bit difference
may flip a convergence test once in a while, which moves the result by at most the slack Ceres' function_tolerance = 1e-6
leaves (<= 2e-4 in pose units, tests/test_pnp_oracle.py) -- allowed for at most 5 % of the problems.  With tight
tolerances both converge to the optimum and must agree to 1e-8 always."""
import numpy as np
import pytest
import torch

from util import pnp_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def po():
    import pnp_oracle
    return pnp_oracle


def _batch(cases):
    f = lambda i: torch.from_numpy(np.stack([c[i] for c in cases])).cuda()   # noqa: E731
    return f(0), f(1), f(2), f(3), f(4)


def test_batch_matches_oracle_default_options(pvb, po):
    cases = [pnp_case(400 + s, pn=9, noise=2.0, pert=(0.3, 0.1) if s % 3 == 0 else (0.05, 0.02)) for s in range(64)]
    uv, p3, W, K, init = _batch(cases)
    rt, info = pvb.uncertainty_pnp_batch(uv, W, p3, K, init, return_info=True)
    rt, info = rt.cpu().numpy(), info.cpu().numpy()
    same = 0
    for i, c in enumerate(cases):
        want, oi = po.uncertainty_pnp(*c[:5], return_info=True)
        if (info[i, 0], info[i, 1]) == (oi["iterations"], oi["termination"]):
            same += 1
            assert np.abs(rt[i] - want).max() < 1e-9, i
        else:
            assert np.abs(rt[i] - want).max() < 2e-4, i
    assert same >= 61


@pytest.mark.parametrize("pn", [5, 9, 17, 40])
def test_tight_tolerances_reach_the_optimum(pvb, po, pn):
    cases = [pnp_case(500 + s, pn=pn, noise=1.5, pert=(0.2, 0.08)) for s in range(8)]
    uv, p3, W, K, init = _batch(cases)
    rt = pvb.uncertainty_pnp_batch(uv, W, p3, K, init, max_num_iterations=200, function_tolerance=1e-16,
                                   gradient_tolerance=1e-14, parameter_tolerance=1e-16).cpu().numpy()
    for i, c in enumerate(cases):
        want = po.uncertainty_pnp(*c[:5], max_num_iterations=200, function_tolerance=1e-16, gradient_tolerance=1e-14,
                                  parameter_tolerance=1e-16)
        assert np.abs(rt[i] - want).max() < 1e-8, (pn, i)


def test_shared_model_points_and_intrinsics(pvb, po):
    """The production shape: one object model and one camera for the whole batch (stride 0), fp32 inputs as the voting
    layer and pvb_uncertainty_weights produce them."""
    base = pnp_case(600, pn=9)
    cases = []
    for s in range(16):
        c = pnp_case(601 + s, pn=9, noise=1.0)
        rng = np.random.default_rng(700 + s)
        # re-project the SHARED model points with this case's pose
        aa, t = c[5][:3], c[5][3:]
        R = po.rodrigues(aa)
        cam = base[1] @ R.T + t
        uv = np.stack([base[3][0, 0] * cam[:, 0] / cam[:, 2] + base[3][0, 2], base[3][1, 1] * cam[:, 1] / cam[:, 2] + base[3][1, 2]], 1)
        uv += rng.normal(size=uv.shape)
        cases.append((uv.astype(np.float32).astype(np.float64), base[1], c[2].astype(np.float32).astype(np.float64), base[3], c[4]))
    uv = torch.from_numpy(np.stack([c[0] for c in cases])).float().cuda()
    W = torch.from_numpy(np.stack([c[2] for c in cases])).float().cuda()
    init = torch.from_numpy(np.stack([c[4] for c in cases])).cuda()
    rt, info = pvb.uncertainty_pnp_batch(uv, W, torch.from_numpy(base[1]).cuda(), torch.from_numpy(base[3]).cuda(), init,
                                         return_info=True)
    rt, info = rt.cpu().numpy(), info.cpu().numpy()
    for i, c in enumerate(cases):
        want, oi = po.uncertainty_pnp(*c, return_info=True)
        tol = 1e-9 if (info[i, 0], info[i, 1]) == (oi["iterations"], oi["termination"]) else 2e-4
        assert np.abs(rt[i] - want).max() < tol, i
    # per-problem copies of the same arrays give the same bits as the shared ones
    rt2 = pvb.uncertainty_pnp_batch(uv, W, torch.from_numpy(base[1]).cuda().expand(16, 9, 3).contiguous(),
                                    torch.from_numpy(base[3]).cuda().expand(16, 3, 3).contiguous(), init)
    assert np.array_equal(rt2.cpu().numpy(), rt)


def test_degenerate_problems_in_a_batch(pvb, po):
    good = pnp_case(800, pn=9)[:5]
    zero_w = (good[0], good[1], np.zeros_like(good[2]), good[3], good[4])
    at_opt = pnp_case(801, pn=9, noise=0.0)
    at_opt = (at_opt[0], at_opt[1], at_opt[2], at_opt[3], at_opt[5])
    nan_w = (good[0], good[1], good[2].copy(), good[3], good[4])
    nan_w[2][2, 0] = np.nan
    behind = (good[0], good[1], good[2], good[3], good[4].copy())
    behind[4][5] = -0.05
    cases = [good, zero_w, at_opt, nan_w, behind]
    uv, p3, W, K, init = _batch(cases)
    rt, info = pvb.uncertainty_pnp_batch(uv, W, p3, K, init, return_info=True)
    rt, info = rt.cpu().numpy(), info.cpu().numpy()
    with np.errstate(all="ignore"):
        want, oi = po.uncertainty_pnp(*good, return_info=True)
    tol = 1e-9 if (info[0, 0], info[0, 1]) == (oi["iterations"], oi["termination"]) else 2e-4   # see the module docstring
    assert np.abs(rt[0] - want).max() < tol
    # all weights zero: every residual and Jacobian entry is exactly 0 -> gradient test at iteration 0, pose untouched
    assert (info[1, 0], info[1, 1]) == (0, po.CONVERGENCE_GRADIENT)
    # started at the optimum of noise-free data: the gradient (~1e-10, the size of the tolerance) decides whether zero or one
    # more iteration is taken, so only the result is pinned
    assert 1 <= info[2, 1] <= 6 and np.abs(rt[2] - at_opt[4]).max() < 1e-8
    # a NaN weight poisons the normal equations: the gradient test is the first to see it, pose untouched
    assert (info[3, 0], info[3, 1]) == (0, po.CONVERGENCE_GRADIENT)
    # points behind the camera: a long, ill-conditioned descent (28 iterations in the oracle) whose path depends on the last
    # bits of the sums -- only required to terminate with a valid code and without touching its neighbours
    assert 1 <= info[4, 1] <= 6 and 0 <= info[4, 0] <= 50
    assert np.array_equal(rt[1], zero_w[4]) and np.array_equal(rt[3], nan_w[4])      # untouched initial poses
    empty = pvb.uncertainty_pnp_batch(uv[:0], W[:0], p3[:0], K[:0], init[:0])
    assert empty.shape == (0, 6)


def test_reference_python_twins(pvb, po):
    """un_pnp_utils.uncertainty_pnp / _v2 twins: OpenCV P3P initialisation exactly as the reference does it, refinement on the
    GPU; compared with the oracle started from the same P3P pose."""
    cv2 = pytest.importorskip("cv2")
    uv, p3, W, K, _, true_rt = pnp_case(900, pn=9, noise=0.5)
    Rt = pvb.un_pnp.uncertainty_pnp(uv, W, p3, K)
    assert Rt.shape == (3, 4)
    idxs = np.argsort(W[:, 0] + W[:, 1])[-4:]
    _, r_exp, t = cv2.solvePnP(np.expand_dims(p3[idxs], 0), np.expand_dims(uv[idxs], 0), K, np.zeros((8, 1)), None, None, False,
                               flags=cv2.SOLVEPNP_P3P)
    want = po.uncertainty_pnp(uv, p3, W, K, np.concatenate([r_exp, t], 0).reshape(6))
    assert np.abs(Rt[:, :3] - po.rodrigues(want[:3])).max() < 1e-6 and np.abs(Rt[:, 3] - want[3:]).max() < 1e-6
    assert np.abs(Rt[:, 3] - true_rt[3:]).max() < 0.05                                   # and it is a sensible pose
    cov = np.stack([np.eye(2) * s for s in np.linspace(0.5, 3.0, 9)])
    Rt2 = pvb.un_pnp.uncertainty_pnp_v2(uv, cov, p3, K)
    assert Rt2.shape == (3, 4) and np.abs(Rt2[:, 3] - true_rt[3:]).max() < 0.05
    Rt4 = pvb.un_pnp.uncertainty_pnp(uv[:4], W[:4], p3[:4], K)                            # pn == 4: the P3P pose itself
    assert Rt4.shape == (3, 4) and np.isfinite(Rt4).all()


def test_input_checks(pvb):
    uv = torch.zeros((2, 9, 2), device="cuda")
    with pytest.raises(RuntimeError):
        pvb.uncertainty_pnp_batch(uv.cpu(), uv, uv, uv, uv)
    with pytest.raises(RuntimeError):
        pvb.uncertainty_pnp_batch(uv, torch.zeros((2, 9, 2), device="cuda"), torch.zeros((9, 3), device="cuda"),
                                  torch.zeros((3, 3), device="cuda"), torch.zeros((2, 6), device="cuda"))
    w = torch.zeros((2, 9, 3), device="cuda")
    for model, cam, name in ((np.zeros((9, 3)), torch.eye(3, device="cuda"), "points_3d"),
                             (torch.zeros((9, 3), device="cuda"), np.eye(3), "camera_matrix")):
        with pytest.raises(RuntimeError, match=f"{name} must be a CUDA tensor"):
            pvb.uncertainty_pnp_batch(uv, w, model, cam, torch.zeros((2, 6), device="cuda"))


def test_kernel_follows_real_ceres(pvb):
    """pvb_uncertainty_pnp against tests/golden/ceres_pnp.npz: 284 problems solved by the reference's own Ceres 2.0 binary
    through its unmodified uncertainty_pnp.cpp (tests/golden/make_golden_ceres.py; CPU counterpart tests/test_ceres_golden.py).
    Same stop reason, same iteration count and the same pose to 1e-9 on the problems an independent implementation can follow
    (`stable`: the result moves < 1e-10 under a 1e-13 perturbation of the start) -- the warp's butterfly sums differ from
    Eigen's in the last bits, which may flip a convergence test on a few of them: then the slack of Ceres' own
    function_tolerance applies (2e-4), for at most 3 %."""
    import os
    G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ceres_pnp.npz"))
    same = total = 0
    for pn in np.unique(G["pn"]):
        idx = np.nonzero(G["pn"] == pn)[0]
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
        rt, info = pvb.uncertainty_pnp_batch(t(G["pts2d"][idx, :pn]), t(G["wgt2d"][idx, :pn]), t(G["pts3d"][idx, :pn]),
                                             t(G["K"][idx]), t(G["init_rt"][idx]), return_info=True)
        rt, info = rt.cpu().numpy(), info.cpu().numpy()
        for j, i in enumerate(idx):
            if G["kind"][i] == "optimum":
                assert np.abs(rt[j] - G["result_rt"][i]).max() < 1e-8, i
                continue
            if not G["stable"][i]:
                assert 1 <= info[j, 1] <= 6, i
                continue
            total += 1
            want_it = int(G["iteration_summaries"][i]) - (0 if G["reason"][i] in (2, 3) else 1)
            if (info[j, 0], info[j, 1]) == (want_it, G["reason"][i]):
                same += 1
                assert np.abs(rt[j] - G["result_rt"][i]).max() < 1e-9, i
            else:
                assert np.abs(rt[j] - G["result_rt"][i]).max() < 2e-4, i
    assert total >= 230 and same >= 0.97 * total, (same, total)


def test_fused_tail_equals_the_three_step_pipeline(pvb):
    """pvb_uncertainty_pnp_from_votes (weights + P3P + LM in one launch, fp32 in) against pvb_uncertainty_weights ->
    pvb_uncertainty_pnp_init -> pvb_uncertainty_pnp on the same data: identical bits, incl. the degenerate covariances the
    reference zeroes (cov[0,0] < 1e-6, NaN) and a problem whose P3P has no admissible pose."""
    n, pn = 40, 9
    cases = [pnp_case(1200 + s, pn=pn, noise=[0.5, 2.0][s % 2]) for s in range(n)]
    rng = np.random.default_rng(5)
    kpt = torch.from_numpy(np.stack([c[0] for c in cases])).float().cuda()
    A = rng.normal(size=(n, pn, 2, 2))
    cov = A @ A.transpose(0, 1, 3, 2) * rng.uniform(0.3, 5.0, size=(n, pn, 1, 1)) + 0.05 * np.eye(2)
    cov[3, 2] = 0.0                       # cov[0,0] < 1e-6 -> weight 0
    cov[4, 5, 0, 1] = np.nan              # NaN -> weight 0
    cov[7, :, :, :] = 0.0                 # every weight 0: P3P still has its 4 points, the LM stops at once on that pose
    cov = torch.from_numpy(cov).float().cuda()
    model = torch.from_numpy(cases[0][1]).cuda()
    cam = torch.from_numpy(cases[0][3]).cuda()
    # re-project the shared model with every case's true pose so the problems are consistent
    from clean_pvnet_b200.uncertainty_pnp import rodrigues
    true = torch.from_numpy(np.stack([c[5] for c in cases])).cuda()
    Rt = rodrigues(true)
    camp = model[None] @ Rt[:, :, :3].transpose(1, 2) + Rt[:, None, :, 3]
    uv = torch.stack([cam[0, 0] * camp[..., 0] / camp[..., 2] + cam[0, 2], cam[1, 1] * camp[..., 1] / camp[..., 2] + cam[1, 2]], -1)
    kpt = (uv + torch.from_numpy(rng.normal(size=(n, pn, 2))).cuda()).float()
    w = pvb.uncertainty_pnp_weights(cov)
    init = pvb.p3p_init_batch(kpt, w, model, cam)
    want, winfo = pvb.uncertainty_pnp_batch(kpt, w, model, cam, init, return_info=True)
    got, info, init_used, w_used = pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, return_info=True, return_aux=True)
    assert torch.equal(w_used, w)
    assert torch.equal(init_used.view(torch.int64), init.view(torch.int64))          # NaN rows included
    assert torch.equal(info, winfo)
    assert torch.equal(got.view(torch.int64), want.view(torch.int64))
    ok = torch.isfinite(got).all(dim=1)
    assert int(ok.sum()) >= n - 3
    assert info[7, 0].item() == 0 and torch.equal(got[7].view(torch.int64), init[7].view(torch.int64))   # zero weights: untouched
    ok[7] = False
    assert (got[ok][:, 3:] - true[ok][:, 3:]).abs().max().item() < 0.08              # and they are sensible poses
    # the weights= form and an explicit init
    got2 = pvb.uncertainty_pnp_from_votes(kpt, None, model, cam, init_rt=init, weights=w)
    assert torch.equal(got2.view(torch.int64), want.view(torch.int64))
    with pytest.raises(RuntimeError):
        pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, weights=w)
