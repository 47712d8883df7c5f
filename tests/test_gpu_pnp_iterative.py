"""GPU: pvb_pnp_iterative / pose.pnp_batch (csrc/pnp.cu pnp_iter_kernel, csrc/pnp_iter_core.cuh), PVNet's default pose step
`cv2.solvePnP(..., SOLVEPNP_ITERATIVE)` for a whole batch:
  - against OpenCV's stored answers (tests/golden/pnp_iterative.npz) at the CPU pin's bar, 1e-8;
  - against the host build of the same core (tests/pnp_iter_host_harness.cpp): the same iterations and statuses, results
    to 1e-10 where the loop converged;
  - batch independence, shared / per-problem model and K, fp32 / fp64 image points, every status code;
  - end to end on a posed synthetic scene: decode_keypoint(un_pnp=False) -> pnp_batch -> linemod_scores gives every
    flag a per-image loop of the reference's pvnet_pose_utils.pnp (OpenCV) and the restated evaluator gives."""
import os

import numpy as np
import pytest
import torch

from pnp_iter_cases import K_LINEMOD, ROOT, STATUS, cases, host_core, rel_diff

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pvb():
    import clean_pvnet_b200 as m
    return m


@pytest.fixture(scope="module")
def core():
    return host_core()


def _fixture():
    F = np.load(os.path.join(ROOT, "tests", "golden", "pnp_iterative.npz"))
    probs = [(F["pts2d"][a:b], F["pts3d"][a:b], F["K"][i], F["rt"][i], F["pose"][i])
             for i, (a, b) in enumerate(zip(F["off"][:-1], F["off"][1:]))]
    return probs, str(F["opencv_version"])


def _device_solve(pts2d, pts3d, K):
    """pvb_pnp_iterative with every output: (pose [n,3,4], rt [n,6], info [n,2]) as numpy"""
    from clean_pvnet_b200.uncertainty_pnp import _call
    p2 = torch.as_tensor(np.ascontiguousarray(pts2d, np.float64)).cuda()
    p3 = torch.as_tensor(np.ascontiguousarray(pts3d, np.float64)).cuda()
    km = torch.as_tensor(np.ascontiguousarray(K, np.float64)).cuda()
    n, pn = p2.shape[:2]
    pose = torch.empty((n, 3, 4), dtype=torch.float64, device="cuda")
    rt = torch.empty((n, 6), dtype=torch.float64, device="cuda")
    info = torch.empty((n, 2), dtype=torch.int32, device="cuda")
    _call("pvb_pnp_iterative", p2.device, p2, p3, km, pose, rt, info, n, pn, 0 if p3.dim() == 2 else pn * 3,
          0 if km.dim() == 2 else 9)
    return pose.cpu().numpy(), rt.cpu().numpy(), info.cpu().numpy()


def _by_pn(probs):
    groups = {}
    for i, p in enumerate(probs):
        groups.setdefault(p[0].shape[0], []).append(i)
    return groups


def test_matches_stored_opencv_and_the_host_core(pvb, core):
    """The host core is built without FMA contraction and sums in point order; nvcc contracts multiply-adds into FMAs and
    the kernel sums by butterfly.  Iteration counts and statuses agree exactly.  Where the loop has converged (status ok)
    the results agree to 1e-10 (1.6e-11 measured on an H100).  A problem stopped by the 20-iteration cap is still moving,
    and the rounding differences grow along its path (1.4e-9 measured): it is held to the OpenCV bar, 1e-8."""
    probs, version = _fixture()
    seen, worst, worst_host = set(), 0.0, {0: 0.0, 1: 0.0}
    for pn, idx in _by_pn(probs).items():
        uv = np.stack([probs[i][0] for i in idx])
        X = np.stack([probs[i][1] for i in idx])
        K = np.stack([probs[i][2] for i in idx])
        pose, rt, info = _device_solve(uv, X, K)
        hpose, hrt, hinfo = core(uv, X, K)
        seen |= set(info[:, 1].tolist())
        for j, i in enumerate(idx):
            d = rel_diff(probs[i][3], rt[j])
            worst = max(worst, d)
            assert d <= 1e-8, (i, pn, d, info[j])
            assert np.abs(pose[j] - probs[i][4]).max() <= 1e-8 * max(1.0, np.abs(probs[i][4]).max()), i
            assert np.array_equal(info[j], hinfo[j]), (i, pn, info[j], hinfo[j])
            st = int(info[j, 1])
            worst_host[st] = max(worst_host[st], rel_diff(hrt[j], rt[j]))
    print(f"\n{len(probs)} problems: within {worst:.2e} of cv2 {version}; of the host core within {worst_host[0]:.2e} "
          f"(ok), {worst_host[1]:.2e} (iteration limit)")
    assert seen == {STATUS["ok"], STATUS["iteration_limit"]}
    assert worst_host[0] <= 1e-10 and worst_host[1] <= 1e-8


def test_batch_independence_and_fp32_points(pvb):
    cs = cases(1000, seed0=5000)
    cs = [c for c in cs if c[0].shape[0] == 9][:1]
    rng = np.random.default_rng(0)
    uv = np.stack([cs[0][0]] * 1000) + rng.normal(size=(1000, 9, 2))
    uv[417] = cs[0][0]
    p2 = torch.from_numpy(uv).cuda()
    big = pvb.pnp_batch(cs[0][1], p2, cs[0][2])
    alone = pvb.pnp_batch(cs[0][1], p2[417:418].clone(), cs[0][2])
    assert torch.equal(big[417], alone[0])
    # a batch of 1000 equals each problem alone, NaN rows included
    p2[3] = float("nan")
    big, info = pvb.pnp_batch(cs[0][1], p2, cs[0][2], return_info=True)
    for i in (0, 3, 999):
        a, ai = pvb.pnp_batch(cs[0][1], p2[i:i + 1].clone(), cs[0][2], return_info=True)
        assert torch.equal(ai[0], info[i]) and np.array_equal(a[0].cpu().numpy(), big[i].cpu().numpy(), equal_nan=True)
    assert int(info[3, 1]) == STATUS["degenerate"]
    # fp32 points are widened exactly (astype(np.float64))
    f32 = p2.float()
    assert torch.equal(pvb.pnp_batch(cs[0][1], f32, cs[0][2]).nan_to_num(7.0),
                       pvb.pnp_batch(cs[0][1], f32.double(), cs[0][2]).nan_to_num(7.0))


@pytest.mark.parametrize("pn", [6, 9, 17, 33, 64])
def test_shared_and_per_problem_model_and_intrinsics(pvb, pn):
    cs = [c for c in cases(600, seed0=9000) if c[0].shape[0] == pn][:8]
    uv = torch.from_numpy(np.stack([c[0] for c in cs])).cuda()
    X0 = cs[0][1]
    per = pvb.pnp_batch(np.repeat(X0[None], len(cs), 0), uv, np.repeat(K_LINEMOD[None], len(cs), 0))
    shared = pvb.pnp_batch(torch.from_numpy(X0).cuda(), uv, torch.from_numpy(K_LINEMOD).cuda())
    assert per.dtype == torch.float64 and per.shape == (len(cs), 3, 4)
    assert np.array_equal(per.cpu().numpy(), shared.cpu().numpy(), equal_nan=True)


def test_every_status_code(pvb):
    rng = np.random.default_rng(4)
    rvec, t = np.array([0.3, -0.2, 0.1]), np.array([0.02, -0.01, 0.8])
    import cv2

    def solve(X, uv):
        pose, info = pvb.pnp_batch(X, torch.from_numpy(np.asarray(uv, np.float64)[None]).cuda(), K_LINEMOD,
                                   return_info=True)
        return pose[0].cpu().numpy(), int(info[0, 1])

    X = rng.uniform(-0.1, 0.1, (9, 3))
    uv = cv2.projectPoints(X, rvec, t, K_LINEMOD, None)[0].reshape(-1, 2)
    pose, st = solve(X, uv)
    assert st == STATUS["ok"] and np.abs(pose[:, 3] - t).max() < 1e-9
    for Xs, u, want in ((X[:5], uv[:5], "too_few_points"), (X[:3], uv[:3], "too_few_points"),
                        (X * [1, 1, 0], cv2.projectPoints(X * [1, 1, 0], rvec, t, K_LINEMOD, None)[0].reshape(-1, 2), "planar"),
                        (X, np.zeros((9, 2)), "degenerate"), (X, np.where(np.arange(18).reshape(9, 2) == 5, np.nan, uv), "degenerate")):
        pose, st = solve(Xs, u)
        assert st == STATUS[want] and np.isnan(pose).all(), want
    probs, _ = _fixture()
    limit = [p for p in probs if p[0].shape[0] == 7]
    _, _, info = _device_solve(np.stack([p[0] for p in limit]), np.stack([p[1] for p in limit]),
                               np.stack([p[2] for p in limit]))
    assert STATUS["iteration_limit"] in info[:, 1].tolist() and (info[info[:, 1] == 1, 0] == 20).all()


def test_numpy_twin(pvb):
    import cv2
    from clean_pvnet_b200.pose import pnp
    uv, X, K = cases(1, seed0=321)[0]
    ref = pvb.pose._reference_pnp(X, uv, K, cv2.SOLVEPNP_ITERATIVE, np.zeros((8, 1)))
    got = pnp(X, uv.astype(np.float32), K)
    assert got.shape == (3, 4) and got.dtype == np.float64
    ref32 = pvb.pose._reference_pnp(X, uv.astype(np.float32), K, cv2.SOLVEPNP_ITERATIVE, np.zeros((8, 1)))
    assert np.abs(got - ref32).max() <= 1e-8 * max(1.0, np.abs(ref32).max())
    assert np.abs(pnp(X, uv, K) - ref).max() <= 1e-8 * max(1.0, np.abs(ref).max())
    # planar models and other methods go to OpenCV as the reference calls it
    Xp = X * [1, 1, 0]
    up = cv2.projectPoints(Xp, np.array([0.2, 0.1, 0.0]), np.array([0.0, 0.0, 0.9]), K, None)[0].reshape(-1, 2)
    assert np.array_equal(pnp(Xp, up, K), pvb.pose._reference_pnp(Xp, up, K, cv2.SOLVEPNP_ITERATIVE, np.zeros((8, 1))))
    assert np.array_equal(pnp(X, uv, K, cv2.SOLVEPNP_EPNP), pvb.pose._reference_pnp(X, uv, K, cv2.SOLVEPNP_EPNP,
                                                                                      np.zeros((8, 1))))


def test_end_to_end_default_config(pvb):
    """decode_keypoint(output, un_pnp=False) (hn 128, max_num 100: the reference's default call) -> pnp_batch ->
    linemod_scores, against a per-image loop of pvnet_pose_utils.pnp (OpenCV) and the restated evaluator on host copies of
    the same kpt_2d."""
    import cv2
    from test_gpu_metrics import _add_mean, _cm_degree_5, _mask_iou, _posed_scene, _proj2d
    B = 6
    model, kpt_3d, pose_gt, Ks, output, mask_gt = _posed_scene(B)
    pose_gt[B - 1, :, 3] += [0.1, 0.0, 0.0]          # one ground truth 10 cm away: its pose metrics all fail
    diameter = float(np.max(np.linalg.norm(model[:, None] - model[None, ::10], axis=-1)))
    pvb.decode_keypoint(output, un_pnp=False, seed=5)
    K = torch.from_numpy(Ks).cuda()
    pose = pvb.pnp_batch(kpt_3d, output["kpt_2d"], K)
    pg = torch.from_numpy(pose_gt).cuda()
    s = pvb.linemod_scores(model, diameter, pose, pg, K, mask_pred=output["mask"], mask_gt=mask_gt)
    kpt_2d, mp, mg = output["kpt_2d"].cpu().numpy(), output["mask"].cpu().numpy(), mask_gt.cpu().numpy()
    want = {"proj2d": [], "add": [], "cmd5": [], "mask_ap": []}
    for i in range(B):
        p = pvb.pose._reference_pnp(kpt_3d, kpt_2d[i], Ks[i], cv2.SOLVEPNP_ITERATIVE, np.zeros((8, 1)))
        assert np.abs(p - pose[i].cpu().numpy()).max() <= 1e-8 * max(1.0, np.abs(p).max()), i
        want["proj2d"].append(bool(_proj2d(model, Ks[i], p, pose_gt[i]) < 5))
        want["add"].append(bool(_add_mean(model, p, pose_gt[i]) < diameter * 0.1))
        t, a = _cm_degree_5(p, pose_gt[i])
        want["cmd5"].append(bool(t < 5 and a < 5))
        want["mask_ap"].append(bool(_mask_iou(mp[i], mg[i]) > 0.7))
    assert {k: v.cpu().numpy().tolist() for k, v in s.items()} == want
    assert want["proj2d"][B - 1] is False and any(want["proj2d"])
