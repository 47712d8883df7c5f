"""PVNet's default pose step on the device: `pnp` of lib/utils/pvnet/pvnet_pose_utils.py:5-38, which both evaluators call once
per image when cfg.test.un_pnp is False (lib/evaluators/linemod/pvnet.py:188, tless_test/pvnet.py:239):

    pnp_batch(points_3d, points_2d, camera_matrix)     n problems in one launch, CUDA tensors in, [n,3,4] poses out
    pnp(points_3d, points_2d, camera_matrix, method)   numpy twin of pvnet_pose_utils.pnp: numpy in, 3x4 [R|t] out

Both run `pvb_pnp_iterative` (csrc/pnp.cu, csrc/pnp_iter_core.cuh): OpenCV's SOLVEPNP_ITERATIVE step for step -- the DLT
start and its 20-iteration Levenberg-Marquardt loop -- pinned against cv2.solvePnP itself (DESIGN.md section 8d).  There is
no CPU implementation behind it.  Planar models (OpenCV's homography start), other methods and non-zero distortion are
not built: `pnp` hands those to OpenCV, `pnp_batch` reports them in `info`.
"""
import numpy as np
import torch

from . import _lib
from .uncertainty_pnp import _batch, _call, _model_camera

STATUS = {_lib.PVB_PNP_OK: "ok", _lib.PVB_PNP_ITERATION_LIMIT: "iteration limit",
          _lib.PVB_PNP_TOO_FEW_POINTS: "too few points", _lib.PVB_PNP_PLANAR: "planar model",
          _lib.PVB_PNP_DEGENERATE: "degenerate"}


def pnp_batch(points_3d, points_2d, camera_matrix, *, return_info=False):
    """cv2.solvePnP(..., SOLVEPNP_ITERATIVE) + [Rodrigues(rvec) | tvec] for n problems in one launch, no host sync.

    points_2d  CUDA tensor [n,pn,2], float32 (decode_keypoint's output['kpt_2d'], widened exactly like the reference's
               astype(np.float64)) or float64
    points_3d  [pn,3] (shared) or [n,pn,3];  camera_matrix [3,3] (shared) or [n,3,3]; tensors or arrays of any float dtype
    Returns pose float64 [n,3,4] on the device of points_2d, which linemod_scores takes as it is; with return_info also
    info int32 [n,2] = (Levenberg-Marquardt iterations, status: 0 ok, 1 iteration limit, 2 too few points, 3 planar
    model, 4 degenerate -- see STATUS).  Every status but 0 and 1 gives an all-NaN pose, which fails every evaluator flag."""
    dev, n, pn = _batch(points_2d, "points_2d")
    if points_2d.dtype not in (torch.float32, torch.float64):
        raise RuntimeError(f"points_2d must be float32 or float64, got {points_2d.dtype}")
    if pn < 1:
        raise RuntimeError("need at least one point per problem")
    p3, km = torch.as_tensor(points_3d), torch.as_tensor(camera_matrix)
    if tuple(p3.shape) not in ((pn, 3), (n, pn, 3)):
        raise RuntimeError(f"points_3d must be [{pn},3] or [{n},{pn},3], got {list(p3.shape)}")
    if tuple(km.shape) not in ((3, 3), (n, 3, 3)):
        raise RuntimeError(f"camera_matrix must be [3,3] or [{n},3,3], got {list(km.shape)}")
    p3, km, s3, sk = _model_camera(p3, km, dev, pn)
    p2 = points_2d.to(torch.float64).contiguous()
    pose = torch.empty((n, 3, 4), dtype=torch.float64, device=dev)
    info = torch.zeros((n, 2), dtype=torch.int32, device=dev) if return_info else None
    if n:
        _call("pvb_pnp_iterative", dev, p2, p3, km, pose, None, info, n, pn, s3, sk)
    return (pose, info) if return_info else pose


def _reference_pnp(points_3d, points_2d, camera_matrix, method, dist_coeffs):
    """pvnet_pose_utils.pnp (:5-38) as the reference runs it, on OpenCV"""
    import cv2
    if method == cv2.SOLVEPNP_EPNP:
        points_3d = np.expand_dims(points_3d, 0)
        points_2d = np.expand_dims(points_2d, 0)
    points_2d = np.ascontiguousarray(points_2d.astype(np.float64))
    points_3d = np.ascontiguousarray(points_3d.astype(np.float64))
    camera_matrix = camera_matrix.astype(np.float64)
    _, R_exp, t = cv2.solvePnP(points_3d, points_2d, camera_matrix, dist_coeffs, flags=method)
    R, _ = cv2.Rodrigues(R_exp)
    return np.concatenate([R, t], axis=-1)


def pnp(points_3d, points_2d, camera_matrix, method=None, device="cuda"):
    """Twin of pvnet_pose_utils.pnp (lib/utils/pvnet/pvnet_pose_utils.py:5-38): points_3d [pn,3], points_2d [pn,2],
    camera_matrix [3,3] numpy arrays in, the float64 3x4 [R | t] out.  method None means cv2.SOLVEPNP_ITERATIVE (the
    reference's default).  ITERATIVE with zero distortion (`pnp.dist_coeffs` unset or all zero, like the reference's
    function attribute) runs on the device; any other method or distortion, and the problems the device reports as planar,
    too few points or degenerate, go to OpenCV exactly as the reference calls it (so they raise or return what it does)."""
    import cv2
    if method is None:
        method = cv2.SOLVEPNP_ITERATIVE
    dist_coeffs = getattr(pnp, "dist_coeffs", None)
    if dist_coeffs is None:
        dist_coeffs = np.zeros(shape=[8, 1], dtype="float64")
    points_3d, points_2d, camera_matrix = np.asarray(points_3d), np.asarray(points_2d), np.asarray(camera_matrix)
    assert points_3d.shape[0] == points_2d.shape[0], "points 3D and points 2D must have same number of vertices"
    if method != cv2.SOLVEPNP_ITERATIVE or np.any(np.asarray(dist_coeffs) != 0) or points_2d.ndim != 2:
        return _reference_pnp(points_3d, points_2d, camera_matrix, method, dist_coeffs)
    dev = torch.device(device)
    p2 = torch.from_numpy(np.ascontiguousarray(points_2d.astype(np.float64)))[None].to(dev)
    pose, info = pnp_batch(points_3d.astype(np.float64), p2, camera_matrix.astype(np.float64), return_info=True)
    if int(info[0, 1]) not in (_lib.PVB_PNP_OK, _lib.PVB_PNP_ITERATION_LIMIT):
        return _reference_pnp(points_3d, points_2d, camera_matrix, method, dist_coeffs)
    return pose[0].cpu().numpy()
