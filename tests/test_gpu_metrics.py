"""The evaluator metrics on the device (pvb_pose_metrics in csrc/nn.cu, pvb_mask_iou in csrc/select.cu, and
clean_pvnet_b200.metrics) against a numpy restatement of what lib/evaluators/linemod/pvnet.py computes per image:

  project         pvnet_pose_utils.py:41-50   camera points = model @ R.T + t, then @ K.T, then xy / z (IEEE division:
                                              z = 0 gives +-inf or NaN, z < 0 projects through the camera centre)
  projection_2d   linemod/pvnet.py:59-66      mean |project(pred) - project(gt)| < 5
  cm_degree_5     pvnet_pose_utils.py:53-60   |t_pred - t_gt| * 100; trace(R_pred R_gt^T) clamped by `trace if trace <= 3
                  (linemod/pvnet.py:84-94)    else 3`, then `trace if trace >= -1 else -1` -- a NaN trace becomes 3, so a
                                              NaN pose gets 0 degrees (and a NaN translation distance); both < 5
  T-LESS          tless_test/pvnet.py:119-125 any pair of (prediction, ground truth) passes cm_degree_5
  mask_iou        linemod/pvnet.py:96-100     (pred & gt).sum() / (pred | gt).sum() over the VALUES of the ops, > 0.7
  add_metric      linemod/pvnet.py:68-82      mean |pred_i - target_i| < self.diameter * 0.1

numpy's 3x3 products go through BLAS, whose use of FMA is not pinned, so the distances are compared to rtol 1e-9 (the bar
ADD uses), and the angle also within 1e-5 degrees where arccos is ill-conditioned (near 0 and 180 degrees)."""
import zlib

import numpy as np
import pytest
import torch

from test_gpu_nn import _rot

pytestmark = pytest.mark.gpu

K_LINEMOD = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])


# ---- numpy restatement ------------------------------------------------------------------------------------------------

def _project(model, K, pose):
    cam = model @ pose[:, :3].T + pose[:, 3]
    img = cam @ K.T
    with np.errstate(divide="ignore", invalid="ignore"):
        return img[:, :2] / img[:, 2:3]


def _proj2d(model, K, pred, gt):
    with np.errstate(invalid="ignore"):
        return np.mean(np.linalg.norm(_project(model, K, pred) - _project(model, K, gt), axis=-1))


def _cm_degree_5(pred, gt):
    trans = np.linalg.norm(pred[:, 3] - gt[:, 3]) * 100
    trace = np.trace(pred[:, :3] @ gt[:, :3].T)
    trace = trace if trace <= 3 else 3
    trace = trace if trace >= -1 else -1
    return trans, np.rad2deg(np.arccos((trace - 1.0) / 2.0))


def _mask_iou(pred, gt):
    with np.errstate(divide="ignore", invalid="ignore"):
        return (pred & gt).sum() / (pred | gt).sum()


def _add_mean(model, pred, gt):
    return np.mean(np.linalg.norm((model @ pred[:, :3].T + pred[:, 3]) - (model @ gt[:, :3].T + gt[:, 3]), axis=-1))


def _close(got, want, rtol=1e-9):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    with np.errstate(invalid="ignore"):                 # inf - inf
        return np.array_equal(np.isnan(got), np.isnan(want)) and bool(np.all(
            (got == want) | np.isnan(want) | (np.abs(got - want) <= rtol * np.abs(want))))


def _angle_close(got, want):
    near_pole = np.minimum(want, 180.0 - want) < 1.0
    return bool(np.all(np.abs(got - want) <= 1e-9 * np.abs(want) + np.where(near_pole, 1e-5, 0.0)))


def _check_pose_metrics(got, model, pred, gt, Ks):
    want = np.array([[_proj2d(model, Ks[i], pred[i], gt[i]), *_cm_degree_5(pred[i], gt[i])] for i in range(len(pred))])
    g = {k: v.cpu().numpy() for k, v in got.items()}
    assert all(v.dtype == np.float64 and v.shape == (len(pred),) for v in g.values())
    assert _close(g["proj2d"], want[:, 0]), np.c_[g["proj2d"], want[:, 0]][:5]
    assert _close(g["trans_cm"], want[:, 1])
    assert _angle_close(g["angle_deg"], want[:, 2]), np.c_[g["angle_deg"], want[:, 2]][:5]
    return want


# ---- poses ------------------------------------------------------------------------------------------------------------

def _turn(rng, deg):
    """A rotation by `deg` degrees about a random axis."""
    k = rng.normal(size=3)
    k /= np.linalg.norm(k)
    S = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    t = np.radians(deg)
    return np.eye(3) + np.sin(t) * S + (1 - np.cos(t)) * S @ S


def _scene(rng, n, pn, per_pair_k):
    """A LINEMOD-sized model (metres) and n pose pairs of three kinds, cycling with the index, built to stay away from the
    5 px / 5 cm / 5 degree thresholds: close (rotated < 1.2 degrees, moved < 0.05 cm), far (moved 10-15 cm), turned
    (rotated 30-170 degrees)."""
    model = rng.normal(size=(pn, 3)) * [0.05, 0.03, 0.04]
    gt = np.concatenate([_rot(rng, n), rng.normal(size=(n, 3, 1)) * [[0.05], [0.05], [0.1]] + [[0], [0], [1.0]]], 2)
    pred = gt.copy()
    kind = np.arange(n) % 3
    small = _rot(rng, n, 0.02)
    for i in range(n):
        pred[i, :, :3] = (_turn(rng, rng.uniform(30, 170)) if kind[i] == 2 else small[i]) @ gt[i, :, :3]
        d = rng.normal(size=3)
        pred[i, :, 3] += d / np.linalg.norm(d) * (rng.uniform(0.1, 0.15) if kind[i] == 1 else rng.uniform(0, 5e-4))
    if per_pair_k:
        Ks = np.repeat(K_LINEMOD[None], n, 0)
        Ks[:, :2] *= rng.uniform(0.9, 1.1, (n, 2, 1))
    else:
        Ks = K_LINEMOD
    return model, pred, gt, Ks


@pytest.mark.parametrize("per_pair_k", [False, True])
@pytest.mark.parametrize("pn", [1, 1000, 20000])
@pytest.mark.parametrize("n", [1, 7, 300])
def test_pose_metrics_match_the_evaluator(pvb, n, pn, per_pair_k):
    rng = np.random.default_rng(n * 7919 + pn + per_pair_k)
    model, pred, gt, Ks = _scene(rng, n, pn, per_pair_k)
    dev = "cuda"
    got = pvb.pose_metrics_batch(torch.from_numpy(model).to(dev), torch.from_numpy(pred).to(dev),
                                 torch.from_numpy(gt).to(dev), torch.from_numpy(Ks).to(dev))
    Kn = Ks if per_pair_k else np.repeat(Ks[None], n, 0)
    want = _check_pose_metrics(got, model, pred, gt, Kn)
    # the flags, on inputs kept away from the thresholds (one model point can sit near a rotation axis)
    assert np.all(np.abs(want[:, 1:] - 5) > 0.5)
    if pn >= 1000:
        assert np.all(np.abs(want[:, 0] - 5) > 0.5)
    diameter = 0.2
    s = pvb.linemod_scores(model, diameter, torch.from_numpy(pred).to(dev), gt, Ks)
    assert set(s) == {"proj2d", "add", "cmd5"} and all(v.dtype == torch.bool and v.is_cuda for v in s.values())
    assert s["proj2d"].cpu().numpy().tolist() == (want[:, 0] < 5).tolist()
    assert s["cmd5"].cpu().numpy().tolist() == ((want[:, 1] < 5) & (want[:, 2] < 5)).tolist()
    add = np.array([_add_mean(model, pred[i], gt[i]) for i in range(n)])
    assert np.all(np.abs(add - diameter * 0.1) > 1e-6)
    assert s["add"].cpu().numpy().tolist() == (add < diameter * 0.1).tolist()
    if n >= 7:                                         # every kind of pair, so both values of every flag
        assert set(s["proj2d"].tolist()) == {True, False} and set(s["cmd5"].tolist()) == {True, False}


def test_pose_metrics_edge_cases(pvb):
    rng = np.random.default_rng(3)
    model, pred, gt, _ = _scene(rng, 6, 500, False)
    I = np.eye(3)
    # identical poses; a NaN pose (the device P3P's failed problem); traces above 3 and below -1
    pred[0] = gt[0]
    pred[1] = np.nan
    pred[2, :, :3] = 1.5 * I; gt[2, :, :3] = I                                  # trace 4.5 -> 0 degrees
    pred[3, :, :3] = -2 * I; gt[3, :, :3] = I                                   # trace -6 -> 180 degrees
    # points on and behind the camera plane: z = 0 gives inf, z < 0 projects through
    gt[4] = np.c_[I, [0.0, 0.0, 0.0]]
    pred[4] = np.c_[I, [0.01, 0.0, 0.5]]
    gt[5] = np.c_[I, [0.0, 0.0, 0.02]]                                          # part of the model is behind z = 0
    pred[5] = np.c_[I, [0.0, 0.0, 0.021]]
    model[0] = [0.1, 0.2, 0.0]
    got = pvb.pose_metrics_batch(model, torch.from_numpy(pred).cuda(), gt, K_LINEMOD)
    want = _check_pose_metrics(got, model, pred, gt, [K_LINEMOD] * 6)
    g = {k: v.cpu().numpy() for k, v in got.items()}
    assert g["proj2d"][0] == 0.0 and g["trans_cm"][0] == 0.0 and g["angle_deg"][0] < 1e-5
    assert g["angle_deg"][1] == 0.0 and np.isnan(g["trans_cm"][1]) and np.isnan(g["proj2d"][1])
    assert g["angle_deg"][2] == 0.0 and abs(g["angle_deg"][3] - 180.0) < 1e-9
    assert g["proj2d"][4] == np.inf and want[4, 0] == np.inf
    assert (model @ gt[5, :, :3].T + gt[5, :, 3])[:, 2].min() < 0 and np.isfinite(want[5, 0])
    s = pvb.linemod_scores(model, 0.2, torch.from_numpy(pred).cuda(), gt, K_LINEMOD)
    assert not s["proj2d"][1] and not s["add"][1] and not s["cmd5"][1]         # the NaN pose fails every test
    assert not s["proj2d"][4] and s["proj2d"][0] and s["cmd5"][0]
    # pn = 0: proj2d is NaN (the mean of nothing), the pose distances are unchanged
    empty = pvb.pose_metrics_batch(np.zeros((0, 3)), torch.from_numpy(pred).cuda(), gt, K_LINEMOD)
    assert torch.isnan(empty["proj2d"]).all()
    for k in ("trans_cm", "angle_deg"):
        assert np.array_equal(empty[k].cpu().numpy(), g[k], equal_nan=True)
    # n = 0
    none = pvb.pose_metrics_batch(model, np.zeros((0, 3, 4)), np.zeros((0, 3, 4)), K_LINEMOD)
    assert all(v.shape == (0,) for v in none.values())


@pytest.mark.parametrize("per_pair_k", [False, True])
def test_pose_metrics_do_not_depend_on_the_batch(pvb, per_pair_k):
    rng = np.random.default_rng(17)
    model, pred, gt, Ks = _scene(rng, 300, 5000, per_pair_k)
    batch = pvb.pose_metrics_batch(model, torch.from_numpy(pred).cuda(), gt, Ks)
    for i in (0, 1, 150, 299):
        one = pvb.pose_metrics_batch(model, torch.from_numpy(pred[i:i + 1]).cuda(), gt[i:i + 1],
                                     Ks[i:i + 1] if per_pair_k else Ks)
        for k in batch:
            assert batch[k][i].cpu().numpy().tobytes() == one[k][0].cpu().numpy().tobytes(), (i, k)


def test_tless_cm_degree_5_is_rows_of_all_pairs(pvb):
    """tless_test/pvnet.py:119-125: an image passes if any (prediction, ground truth) pair passes."""
    rng = np.random.default_rng(23)
    seen = set()
    for trial in range(6):
        npred, ngt = 1 + trial % 3, 1 + (trial * 5) % 4
        model, pred, gt, _ = _scene(rng, 3 * max(npred, ngt), 200, False)
        rows = np.arange(len(pred))
        # even trials: close predictions, one of which meets its ground truth; odd trials: far ones, which match none
        pidx = rows[rows % 3 == trial % 2][:npred]
        P, G = pred[pidx], gt[np.r_[pidx[-1], rows[rows % 3 == 2]][:ngt]]
        m = pvb.pose_metrics_batch(model, torch.from_numpy(np.repeat(P, ngt, 0)).cuda(), np.tile(G, (npred, 1, 1)),
                                   K_LINEMOD)
        got = bool(((m["trans_cm"] < 5) & (m["angle_deg"] < 5)).any())
        want = False
        for p in P:
            for g in G:
                t, a = _cm_degree_5(p, g)
                if t < 5 and a < 5:
                    want = True
        assert got == want, trial
        seen.add(got)
    assert seen == {True, False}


# ---- mask IoU -----------------------------------------------------------------------------------------------------------

def _mask(g, dtype, B, H, W):
    if dtype == torch.bool:
        return torch.rand((B, H, W), generator=g) < 0.4
    if dtype == torch.int8:                                    # negative values too
        return torch.randint(-128, 128, (B, H, W), generator=g, dtype=torch.int16).to(torch.int8)
    if dtype == torch.uint8:                                   # a 0 / 1 / 255 ground truth
        v = torch.randint(0, 3, (B, H, W), generator=g)
        return torch.where(v == 2, 255, v).to(torch.uint8)
    return torch.randint(0, 4, (B, H, W), generator=g).to(dtype)   # class indices above 1


def _check_iou(pvb, pred, gt):
    inter, uni = pvb.metrics._mask_iou_sums(pred, gt)
    iou = pvb.mask_iou_batch(pred, gt).cpu().numpy()
    p, g = pred.cpu().numpy(), gt.cpu().numpy()
    for b in range(p.shape[0]):
        assert int(inter[b]) == int((p[b] & g[b]).sum()), b
        assert int(uni[b]) == int((p[b] | g[b]).sum()), b
        want = _mask_iou(p[b], g[b])
        assert (np.isnan(iou[b]) and np.isnan(want)) or iou[b] == want, (b, iou[b], want)
    return iou


@pytest.mark.parametrize("pd", [torch.int64, torch.int32, torch.uint8, torch.bool])
@pytest.mark.parametrize("gd", [torch.uint8, torch.bool, torch.int64, torch.int8])
def test_mask_iou_dtypes(pvb, pd, gd):
    g = torch.Generator().manual_seed(zlib.crc32(f"{pd} {gd}".encode()))
    _check_iou(pvb, _mask(g, pd, 2, 480, 640).cuda(), _mask(g, gd, 2, 480, 640).cuda())


@pytest.mark.parametrize("B,H,W", [(1, 480, 640), (16, 480, 640), (64, 480, 640), (3, 479, 641), (2, 7, 5), (1, 1, 1)])
def test_mask_iou_shapes(pvb, B, H, W):
    g = torch.Generator().manual_seed(B * 1000 + H + W)
    _check_iou(pvb, _mask(g, torch.int64, B, H, W).cuda(), _mask(g, torch.uint8, B, H, W).cuda())


def test_mask_iou_views(pvb):
    g = torch.Generator().manual_seed(99)
    B, H, W = 4, 480, 640
    pred = _mask(g, torch.int64, B, W, H).cuda().permute(0, 2, 1)                     # permuted: x stride H
    gt = _mask(g, torch.uint8, B, H + 5, W + 9).cuda()[:, 2:2 + H, 4:4 + W]           # sliced rows
    assert not pred.is_contiguous() and not gt.is_contiguous()
    _check_iou(pvb, pred, gt)
    every_other = _mask(g, torch.int64, 2 * B, H, W).cuda()[::2]                      # contiguous images, batch stride 2HW
    _check_iou(pvb, every_other, _mask(g, torch.uint8, B, H, W).cuda())
    flat = _mask(g, torch.int64, 1, 1, B * H * W + 1).cuda().view(-1)                  # images not 16-byte aligned
    _check_iou(pvb, flat[1:].view(B, H, W), _mask(g, torch.bool, B, H, W).cuda())
    _check_iou(pvb, pred, gt.to(torch.int8))


def test_mask_iou_empty_union_and_two_class_values(pvb):
    z = torch.zeros((3, 48, 64), dtype=torch.int64, device="cuda")
    gt = torch.zeros((3, 48, 64), dtype=torch.uint8, device="cuda")
    z[1, :10] = 2                                                                      # 2 & 1 = 0, 2 | 1 = 3
    gt[1, :20] = 1
    z[2, :4] = 1
    gt[2, 2:6] = 255                                                                   # 1 & 255 = 1, 1 | 255 = 255
    iou = _check_iou(pvb, z, gt)
    assert np.isnan(iou[0])
    inter, uni = pvb.metrics._mask_iou_sums(z, gt)
    assert inter.tolist() == [0, 0, 2 * 64] and uni.tolist() == [0, 10 * 64 * 3 + 10 * 64, 2 * 64 + 2 * 64 * 255 + 2 * 64 * 255]


def test_mask_iou_rejects_floats(pvb):
    with pytest.raises(RuntimeError, match="float"):
        pvb.mask_iou_batch(torch.zeros((1, 4, 4), device="cuda"), torch.zeros((1, 4, 4), dtype=torch.uint8, device="cuda"))


# ---- end to end -------------------------------------------------------------------------------------------------------

def _posed_scene(B, H=480, W=640, seed=0):
    """Synthetic network outputs of B posed views of one random model: seg logits from a mask around the projected object,
    a noisy unit-vector field pointing at the projected keypoints (compute_vertex, pvnet_data_utils.py:30-44, as synth.py
    does for 2-D keypoints), and a ground-truth mask perturbed from the predicted one."""
    rng = np.random.default_rng(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    model = rng.normal(size=(3000, 3)) * [0.04, 0.03, 0.035]
    kpt_3d = np.concatenate([model[rng.choice(len(model), 8, replace=False)], model.mean(0, keepdims=True)])
    pose_gt = np.concatenate([_rot(rng, B, 0.6), np.stack([rng.uniform(-0.08, 0.08, B), rng.uniform(-0.06, 0.06, B),
                                                           rng.uniform(0.7, 1.0, B)], 1)[:, :, None]], 2)
    Ks = np.repeat(K_LINEMOD[None], B, 0)
    yy = torch.arange(H, device="cuda", dtype=torch.float32)[:, None]
    xx = torch.arange(W, device="cuda", dtype=torch.float32)[None, :]
    segs, verts, gts = [], [], []
    for b in range(B):
        kp = torch.from_numpy(_project(kpt_3d, Ks[b], pose_gt[b])).float().cuda()
        pts = _project(model, Ks[b], pose_gt[b])
        c = pts.mean(0)
        r = np.percentile(np.linalg.norm(pts - c, axis=1), 90)
        m = (xx - float(c[0])) ** 2 + (yy - float(c[1])) ** 2 <= r * r
        seg1 = torch.where(m, 2.0, -2.0) + torch.rand((H, W), generator=g, device="cuda") * 0.5
        segs.append(torch.stack([torch.zeros_like(seg1), seg1]))
        ang = torch.atan2(kp[None, None, :, 1] - yy[..., None], kp[None, None, :, 0] - xx[..., None])
        ang = ang + torch.randn(ang.shape, generator=g, device="cuda") * np.radians(2.0)
        verts.append(torch.stack([torch.cos(ang), torch.sin(ang)], -1).reshape(H, W, 18).permute(2, 0, 1))
        # b % 3 == 2: a ground-truth mask of a third of the area (IoU < 0.7); otherwise shifted by two pixels
        rg = r * (0.55 if b % 3 == 2 else 1.0)
        gts.append(((xx - float(c[0]) - 2) ** 2 + (yy - float(c[1])) ** 2 <= rg * rg).to(torch.uint8))
    out = {"seg": torch.stack(segs).contiguous(), "vertex": torch.stack(verts).contiguous()}
    return model, kpt_3d, pose_gt, Ks, out, torch.stack(gts)


def test_end_to_end_linemod_scores(pvb):
    from clean_pvnet_b200.uncertainty_pnp import rodrigues
    B = 6
    model, kpt_3d, pose_gt, Ks, output, mask_gt = _posed_scene(B)
    pose_gt[B - 1, :, 3] += [0.1, 0.0, 0.0]          # one ground truth 10 cm away: its pose metrics all fail
    diameter = float(np.max(np.linalg.norm(model[:, None] - model[None, ::10], axis=-1)))
    pvb.decode_keypoint(output, un_pnp=True, seed=5)
    K = torch.from_numpy(Ks).cuda()
    rt = pvb.uncertainty_pnp_from_votes(output["kpt_2d"], output["var"], torch.from_numpy(kpt_3d).cuda(), K)
    pose = rodrigues(rt)
    pg = torch.from_numpy(pose_gt).cuda()
    for syn in (False, True):
        s = pvb.linemod_scores(model, diameter, pose, pg, K, syn=syn, mask_pred=output["mask"], mask_gt=mask_gt)
        assert set(s) == {"proj2d", "add", "cmd5", "mask_ap"}
        assert all(v.is_cuda and v.dtype == torch.bool and v.shape == (B,) for v in s.values())
        add = pvb.add_metric_batch(model, pose, pg, syn)
        assert torch.equal(s["add"], add < diameter * 0.1)
        if syn:
            continue
        p, mp, mg = pose.cpu().numpy(), output["mask"].cpu().numpy(), mask_gt.cpu().numpy()
        want = {"proj2d": [], "add": [], "cmd5": [], "mask_ap": []}
        for i in range(B):
            want["proj2d"].append(bool(_proj2d(model, Ks[i], p[i], pose_gt[i]) < 5))
            want["add"].append(bool(_add_mean(model, p[i], pose_gt[i]) < diameter * 0.1))
            t, a = _cm_degree_5(p[i], pose_gt[i])
            want["cmd5"].append(bool(t < 5 and a < 5))
            want["mask_ap"].append(bool(_mask_iou(mp[i], mg[i]) > 0.7))
        assert {k: v.cpu().numpy().tolist() for k, v in s.items()} == want
        assert all(set(v) == {True, False} for v in want.values()), want      # both outcomes of every metric occur
        assert np.isclose(add.cpu().numpy(), [_add_mean(model, p[i], pose_gt[i]) for i in range(B)], rtol=1e-9,
                          atol=0).all()
