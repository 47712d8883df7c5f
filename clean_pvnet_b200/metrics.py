"""The LINEMOD evaluator's per-image metrics for a whole batch on the device (lib/evaluators/linemod/pvnet.py:175-205
appends four booleans per image; ADD / ADD-S is `nn.add_metric_batch`):

    pose_metrics_batch(model, pose_pred, pose_gt, K)     projection_2d (:59-66) and cm_degree_5 (:84-94) distances of n
                                                         pose pairs -> dict of float64 [n] tensors
    mask_iou_batch(mask_pred, mask_gt)                   mask_iou (:96-100) of B images -> float64 [B]
    linemod_scores(model, diameter, pose_pred, ...)      the four flags Evaluator.evaluate appends, as bool [n] tensors

T-LESS's cm_degree_5_metric (tless_test/pvnet.py:119-125: any of all (prediction, ground truth) pairs) is the caller
expanding its pairs into rows of pose_metrics_batch, as adi_metric does with add_metric_batch.  Nothing is copied to the
host: the poses and masks stay on the device, and every result is a CUDA tensor.
"""
import ctypes

import torch

from . import _lib
from .nn import _call, _workspace, add_metric_batch

# torch dtype -> pvb_mask_dtype; bool is stored as one byte holding 0 or 1
_MASK_DTYPES = {torch.bool: _lib.PVB_MASK_U8, torch.uint8: _lib.PVB_MASK_U8, torch.int8: _lib.PVB_MASK_I8,
                torch.int16: _lib.PVB_MASK_I16, torch.int32: _lib.PVB_MASK_I32, torch.int64: _lib.PVB_MASK_I64}


def _pose_inputs(model, pose_pred, pose_gt, K):
    """(device, model, pose_pred, pose_gt, K, k_stride) as contiguous float64 on the device of pose_pred (the current
    CUDA device when it is not a CUDA tensor); raises RuntimeError on a bad shape, before anything moves."""
    m, pp, pg, km = (torch.as_tensor(t) for t in (model, pose_pred, pose_gt, K))
    if m.dim() != 2 or m.shape[1] != 3:
        raise RuntimeError(f"model must be [pn,3], got {list(m.shape)}")
    if pp.dim() != 3 or tuple(pp.shape[1:]) != (3, 4) or pp.shape != pg.shape:
        raise RuntimeError(f"pose_pred and pose_gt must both be [n,3,4], got {list(pp.shape)} and {list(pg.shape)}")
    n = int(pp.shape[0])
    if tuple(km.shape) not in ((3, 3), (n, 3, 3)):
        raise RuntimeError(f"K must be [3,3] or [{n},3,3], got {list(km.shape)}")
    dev = pp.device if pp.is_cuda else torch.device("cuda", torch.cuda.current_device())
    f64 = lambda t: t.to(device=dev, dtype=torch.float64).contiguous()   # noqa: E731
    return dev, f64(m), f64(pp), f64(pg), f64(km), 0 if km.dim() == 2 else 9


def _launch_pose_metrics(dev, m, pp, pg, km, k_stride):
    n, pn = int(pp.shape[0]), int(m.shape[0])
    out = {k: torch.empty(n, dtype=torch.float64, device=dev) for k in ("proj2d", "trans_cm", "angle_deg")}
    nbytes = _lib.load().pvb_pose_metrics_workspace_bytes(n, pn)
    _call("pvb_pose_metrics", dev, m, pp, pg, km, k_stride, out["proj2d"], out["trans_cm"], out["angle_deg"], n, pn,
          _workspace(nbytes, dev), nbytes)
    return out


def pose_metrics_batch(model, pose_pred, pose_gt, K):
    """The distances behind Evaluator.projection_2d and cm_degree_5_metric (lib/evaluators/linemod/pvnet.py:59-66, 84-94)
    for n pose pairs at once: model [pn,3] (shared), pose_pred / pose_gt [n,3,4] ([R|t]), K [3,3] or [n,3,3]; tensors or
    arrays, computed in float64.  Returns dict(proj2d=, trans_cm=, angle_deg=), each float64 [n] on the device of
    pose_pred (the current CUDA device when it is not a CUDA tensor):
        proj2d     mean |project(model, K, pred) - project(model, K, gt)| in pixels (pvnet_pose_utils.project: points at
                   z <= 0 give what IEEE division gives, so the mean is inf or NaN; pn = 0 gives NaN)
        trans_cm   |t_pred - t_gt| * 100
        angle_deg  rad2deg(arccos((trace - 1) / 2)) of trace(R_pred R_gt^T), clamped to [-1, 3] by the reference's
                   comparisons, so a NaN pose (the device P3P's failed problem) gets 0 degrees and a NaN trans_cm.
    Compare with the thresholds yourself (< 5 pixels; < 5 cm and < 5 degrees), or call linemod_scores.  For T-LESS's
    cm_degree_5_metric, put every (prediction, ground truth) pair of an image in a row and take any() of its flags."""
    return _launch_pose_metrics(*_pose_inputs(model, pose_pred, pose_gt, K))


def _mask_inputs(mask_pred, mask_gt):
    """Checks two [B,H,W] integer or bool CUDA tensors on one device; raises RuntimeError otherwise."""
    if not (isinstance(mask_pred, torch.Tensor) and isinstance(mask_gt, torch.Tensor) and mask_pred.is_cuda and
            mask_gt.is_cuda):
        raise RuntimeError("mask_pred and mask_gt must be CUDA tensors")
    if mask_pred.device != mask_gt.device:
        raise RuntimeError(f"mask_pred and mask_gt must be on one device, got {mask_pred.device} and {mask_gt.device}")
    if mask_pred.dim() != 3 or mask_pred.shape != mask_gt.shape:
        raise RuntimeError(f"mask_pred and mask_gt must both be [B,H,W], got {list(mask_pred.shape)} and "
                           f"{list(mask_gt.shape)}")
    for name, t in (("mask_pred", mask_pred), ("mask_gt", mask_gt)):
        if t.dtype not in _MASK_DTYPES:
            raise RuntimeError(f"{name} must be a bool or signed integer / uint8 tensor (numpy's `&` takes no floats), "
                               f"got {t.dtype}")


def _mask_iou_sums(mask_pred, mask_gt):
    """(inter, uni): int64 [B] sums of the values of mask_pred & mask_gt and mask_pred | mask_gt, per image."""
    _mask_inputs(mask_pred, mask_gt)
    dev = mask_pred.device
    B, H, W = (int(s) for s in mask_pred.shape)
    inter = torch.empty(B, dtype=torch.int64, device=dev)
    uni = torch.empty(B, dtype=torch.int64, device=dev)
    stride = lambda t: (ctypes.c_int64 * 3)(*t.stride())   # noqa: E731
    p = mask_pred.data_ptr() or None
    g = mask_gt.data_ptr() or None
    _call("pvb_mask_iou", dev, ctypes.c_void_p(p), _MASK_DTYPES[mask_pred.dtype], stride(mask_pred), ctypes.c_void_p(g),
          _MASK_DTYPES[mask_gt.dtype], stride(mask_gt), inter, uni, B, H, W)
    return inter, uni


def mask_iou_batch(mask_pred, mask_gt):
    """Evaluator.mask_iou (lib/evaluators/linemod/pvnet.py:96-100) for B images at once, without the host copies:
    (mask_pred & mask_gt).sum() / (mask_pred | mask_gt).sum() per image, with the sums taken over the VALUES of the
    bitwise ops like numpy (with more than two classes, 2 & 1 = 0 and 2 | 1 = 3).  mask_pred / mask_gt: [B,H,W] CUDA
    tensors of bool, uint8, int8, int16, int32 or int64, any strides (decode_keypoint's int64 output['mask'], which is
    the argmax(seg) the evaluator recomputes, and batch['mask']).  Returns float64 [B]; an empty union gives NaN."""
    inter, uni = _mask_iou_sums(mask_pred, mask_gt)
    return inter.to(torch.float64) / uni.to(torch.float64)


def linemod_scores(model, diameter, pose_pred, pose_gt, K, syn=False, mask_pred=None, mask_gt=None):
    """The booleans Evaluator.evaluate (lib/evaluators/linemod/pvnet.py:175-205) appends for n images, with its own
    thresholds and comparison forms, as bool [n] CUDA tensors:
        proj2d   projection_2d:      proj2d < 5                                 (:59-66)
        add      add_metric:         mean_dist < diameter * 0.1                 (:68-82; syn=True for eggbox and glue)
        cmd5     cm_degree_5_metric: trans_cm < 5 and angle_deg < 5             (:84-94)
        mask_ap  mask_iou:           iou > 0.7, only when both masks are given  (:96-100)
    model [pn,3], pose_pred / pose_gt [n,3,4], K [3,3] or [n,3,3] as in pose_metrics_batch; diameter is the evaluator's
    self.diameter (metres); mask_pred / mask_gt [n,H,W] as in mask_iou_batch.  Every input is checked before any launch."""
    if (mask_pred is None) != (mask_gt is None):
        raise RuntimeError("pass both mask_pred and mask_gt, or neither")
    args = _pose_inputs(model, pose_pred, pose_gt, K)
    if mask_pred is not None:
        _mask_inputs(mask_pred, mask_gt)
        if mask_pred.shape[0] != args[2].shape[0]:
            raise RuntimeError(f"one mask per pose pair: {args[2].shape[0]} pairs, {mask_pred.shape[0]} masks")
    threshold = float(diameter) * 0.1                      # self.diameter * percentage, a Python float
    pm = _launch_pose_metrics(*args)
    out = {"proj2d": pm["proj2d"] < 5,
           "add": add_metric_batch(args[1], args[2], args[3], syn) < threshold,
           "cmd5": (pm["trans_cm"] < 5) & (pm["angle_deg"] < 5)}
    if mask_pred is not None:
        out["mask_ap"] = mask_iou_batch(mask_pred, mask_gt) > 0.7
    return out
