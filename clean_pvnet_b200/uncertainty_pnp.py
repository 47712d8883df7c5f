"""Twins of `lib/csrc/uncertainty_pnp/un_pnp_utils.py` with the Ceres solve replaced by the batched CUDA refinement
(`pvb_uncertainty_pnp`, csrc/pnp.cu; SURVEY.md section 8f row 3).

    uncertainty_pnp(points_2d, weights_2d, points_3d, camera_matrix)        un_pnp_utils.py:6-57
    uncertainty_pnp_v2(points_2d, covars, points_3d, camera_matrix)         un_pnp_utils.py:60-121
    uncertainty_pnp_batch(...)                                              n problems in one launch, CUDA tensors in/out
    p3p_init_batch(...)                                                     the P3P initial poses for a batch, on the device
    uncertainty_pnp_from_votes(kpt_2d, var, ...)                            weights + P3P + refinement in ONE launch, fp32 in

The numpy twins keep the reference's initial pose: OpenCV P3P on the 4 best-weighted points (`cv2.solvePnP(..., SOLVEPNP_P3P)`,
un_pnp_utils.py:27-31) on the host, or an `init_rt` you pass (the pose of a plain PnP, of the previous frame, ...).  The
batched entry can also take it from `p3p_init_batch` -- the same recipe on the device (csrc/p3p_core.cuh, pinned against
cv2.solvePnP on the CPU and on the GPU box).  The refinement runs on the GPU in fp64 with Ceres 2.0's default
Levenberg-Marquardt loop, pinned against the reference's own Ceres binary (tests/golden/ceres_pnp.npz); there is no CPU
implementation behind it.
"""
import ctypes

import numpy as np
import torch

from . import _lib


def _options(max_num_iterations, function_tolerance, gradient_tolerance, parameter_tolerance):
    o = _lib.PvbPnpOptions()
    o.max_num_iterations, o.reserved = int(max_num_iterations), 0
    o.function_tolerance, o.gradient_tolerance = float(function_tolerance), float(gradient_tolerance)
    o.parameter_tolerance = float(parameter_tolerance)
    return ctypes.cast(ctypes.pointer(o), ctypes.c_void_p)


def _batch(points_2d, name):
    """The first check of the three batched entries: `points_2d` must be a CUDA tensor [n,pn,2].  Returns (device, n, pn)."""
    if not (isinstance(points_2d, torch.Tensor) and points_2d.is_cuda):
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if points_2d.dim() != 3 or points_2d.shape[-1] != 2:
        raise RuntimeError(f"{name} must be [n,pn,2]")
    return points_2d.device, int(points_2d.shape[0]), int(points_2d.shape[1])


def _model_camera(points_3d, camera_matrix, dev, pn):
    """The model points ([pn,3] for the whole batch, or [n,pn,3]) and the camera ([3,3] or [n,3,3]), already checked by
    the entry, as float64 on `dev`, with the strides the C entries take (0: shared)."""
    p3 = points_3d.to(device=dev, dtype=torch.float64).contiguous()
    km = camera_matrix.to(device=dev, dtype=torch.float64).contiguous()
    return p3, km, 0 if p3.dim() == 2 else pn * 3, 0 if km.dim() == 2 else 9


def _call(entry, dev, *args):
    """lib.<entry>(*args, stream) on the current stream of `dev`; tensors go in as their device pointers, None as NULL."""
    lib = _lib.load()
    args = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        _lib.check(getattr(lib, entry)(*args, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))


def uncertainty_pnp_batch(points_2d, weights_2d, points_3d, camera_matrix, init_rt=None, *, max_num_iterations=50,
                          function_tolerance=1e-6, gradient_tolerance=1e-10, parameter_tolerance=1e-8, return_info=False):
    """points_2d [n,pn,2], weights_2d [n,pn,3] (wxx,wxy,wyy), points_3d [pn,3] or [n,pn,3], camera_matrix [3,3] or [n,3,3],
    init_rt [n,6] (angle-axis, translation): CUDA tensors of any float dtype.  Returns result_rt [n,6] float64 on the same
    device (and info [n,2] int32 = iterations, termination code when return_info).  Stream-ordered, no host sync.
    init_rt=None: the initial poses come from `p3p_init_batch` (the reference's P3P recipe, on the device)."""
    dev, n, pn = _batch(points_2d, "points_2d")
    if pn < 1:
        raise RuntimeError("need at least one point per problem")

    def check(t, shape, name):
        if not (isinstance(t, torch.Tensor) and t.device == dev):
            raise RuntimeError(f"{name} must be a CUDA tensor on {dev}")
        if tuple(t.shape) != shape:
            raise RuntimeError(f"{name} must have shape {list(shape)}, got {list(t.shape)}")

    f64 = lambda t: t.to(torch.float64).contiguous()   # noqa: E731
    check(points_2d, (n, pn, 2), "points_2d")
    check(weights_2d, (n, pn, 3), "weights_2d")
    shared = lambda t: isinstance(t, torch.Tensor) and t.dim() == 2   # noqa: E731
    check(points_3d, (pn, 3) if shared(points_3d) else (n, pn, 3), "points_3d")
    check(camera_matrix, (3, 3) if shared(camera_matrix) else (n, 3, 3), "camera_matrix")
    if init_rt is not None:
        check(init_rt, (n, 6), "init_rt")
    p2, w2 = f64(points_2d), f64(weights_2d)
    p3, km, s3, sk = _model_camera(points_3d, camera_matrix, dev, pn)
    rt0 = f64(init_rt) if init_rt is not None else p3p_init_batch(p2, w2, p3, km)
    out = torch.empty((n, 6), dtype=torch.float64, device=dev)
    info = torch.zeros((n, 2), dtype=torch.int32, device=dev) if return_info else None
    if n:
        _call("pvb_uncertainty_pnp", dev, p2, p3, w2, km, rt0, out, info, n, pn, s3, sk,
              _options(max_num_iterations, function_tolerance, gradient_tolerance, parameter_tolerance))
    return (out, info) if return_info else out


def uncertainty_pnp_from_votes(kpt_2d, var, points_3d, camera_matrix, init_rt=None, *, weights=None, max_num_iterations=50,
                               function_tolerance=1e-6, gradient_tolerance=1e-10, parameter_tolerance=1e-8,
                               return_info=False, return_aux=False):
    """The evaluator's whole un_pnp tail in ONE launch, straight from the voting layer's outputs (SURVEY 8f rows 2+3):

        kpt_2d [n,pn,2] float32, var [n,pn,2,2] float32  = decode_keypoint's output['kpt_2d'], output['var']
        -> weights = inv(sqrtm(var))            (lib/evaluators/linemod/pvnet.py:118-130, a scipy loop per keypoint)
        -> P3P on the four best-weighted points  (un_pnp_utils.py:25-31, OpenCV on the CPU)       [unless init_rt is given]
        -> Levenberg-Marquardt refinement        (un_pnp_utils.py:49-53 -> Ceres on the CPU)
        -> result_rt [n,6] float64 (angle-axis, translation) on the same device; `rodrigues()` turns it into [n,3,4].

    points_3d [pn,3] or [n,pn,3], camera_matrix [3,3] or [n,3,3] (any float dtype; converted to float64 once).  Pass
    `weights` [n,pn,3] float32 instead of `var` (var=None) if they already exist.  Bit-identical to
    uncertainty_pnp_weights -> p3p_init_batch -> uncertainty_pnp_batch.  No host sync.
    return_info: also info [n,2] int32 (iterations, termination code); return_aux: also (init_rt used, weights)."""
    dev, n, pn = _batch(kpt_2d, "kpt_2d")
    if (var is None) == (weights is None):
        raise RuntimeError("pass exactly one of var / weights")
    k2 = kpt_2d.float().contiguous()
    cv = wt = None
    if var is not None:
        if tuple(var.shape) != (n, pn, 2, 2) or var.device != dev:
            raise RuntimeError(f"var must be a CUDA tensor [{n},{pn},2,2] on {dev}")
        cv = var.float().contiguous()
    else:
        if tuple(weights.shape) != (n, pn, 3) or weights.device != dev:
            raise RuntimeError(f"weights must be a CUDA tensor [{n},{pn},3] on {dev}")
        wt = weights.float().contiguous()
    if tuple(points_3d.shape[-2:]) != (pn, 3) or tuple(camera_matrix.shape[-2:]) != (3, 3):
        raise RuntimeError("points_3d must be [pn,3] | [n,pn,3] and camera_matrix [3,3] | [n,3,3]")
    p3, km, s3, sk = _model_camera(points_3d, camera_matrix, dev, pn)
    rt0 = None
    if init_rt is not None:
        if tuple(init_rt.shape) != (n, 6):
            raise RuntimeError("init_rt must be [n,6]")
        rt0 = init_rt.to(device=dev, dtype=torch.float64).contiguous()
    out = torch.empty((n, 6), dtype=torch.float64, device=dev)
    info = torch.zeros((n, 2), dtype=torch.int32, device=dev) if return_info else None
    init_out = torch.empty((n, 6), dtype=torch.float64, device=dev) if return_aux else None
    w_out = torch.empty((n, pn, 3), dtype=torch.float32, device=dev) if return_aux else None
    if n:
        _call("pvb_uncertainty_pnp_from_votes", dev, k2, cv, wt, p3, km, rt0, out, init_out, w_out, info, n, pn, s3, sk,
              _options(max_num_iterations, function_tolerance, gradient_tolerance, parameter_tolerance))
    res = (out,)
    if return_info:
        res += (info,)
    if return_aux:
        res += (init_out, w_out)
    return res if len(res) > 1 else out


def p3p_init_batch(points_2d, weights_2d, points_3d, camera_matrix):
    """Initial poses [n,6] as un_pnp_utils.py:25-31 computes them with OpenCV (P3P on the 2nd..4th best-weighted keypoints by
    wxx+wxy, the best one picks the root), on the device and for the whole batch; NaN rows where no pose is admissible.
    Pinned against cv2.solvePnP on the CPU (tests/test_p3p_host_core.py) and on the GPU (tests/test_gpu_zz_p3p.py)."""
    dev, n, pn = _batch(points_2d, "points_2d")
    if tuple(weights_2d.shape) != (n, pn, 3) or tuple(points_3d.shape[-2:]) != (pn, 3) or tuple(camera_matrix.shape[-2:]) != (3, 3):
        raise RuntimeError("shapes: points_2d [n,pn,2], weights_2d [n,pn,3], points_3d [pn,3]|[n,pn,3], camera_matrix [3,3]|[n,3,3]")
    if pn < 4:
        raise RuntimeError("the P3P initialisation needs at least 4 points per problem")
    p3, km, s3, sk = _model_camera(points_3d, camera_matrix, dev, pn)
    p2 = points_2d.to(torch.float64).contiguous()
    w2 = weights_2d.to(device=dev, dtype=torch.float64).contiguous()
    out = torch.empty((n, 6), dtype=torch.float64, device=dev)
    if n:
        _call("pvb_uncertainty_pnp_init", dev, p2, p3, w2, km, out, n, pn, s3, sk)
    return out


def rodrigues(rt):
    """[n,6] (angle-axis, translation) -> [n,3,4] (R | t), the conversion un_pnp_utils.py:55-56 does with cv2.Rodrigues."""
    aa, t = rt[..., :3], rt[..., 3:]
    theta = aa.norm(dim=-1, keepdim=True)
    safe = theta.clamp_min(1e-300)
    w = aa / safe
    c, s = torch.cos(theta)[..., None], torch.sin(theta)[..., None]
    wx = torch.zeros(aa.shape[:-1] + (3, 3), dtype=rt.dtype, device=rt.device)
    wx[..., 0, 1], wx[..., 0, 2] = -w[..., 2], w[..., 1]
    wx[..., 1, 0], wx[..., 1, 2] = w[..., 2], -w[..., 0]
    wx[..., 2, 0], wx[..., 2, 1] = -w[..., 1], w[..., 0]
    eye = torch.eye(3, dtype=rt.dtype, device=rt.device).expand_as(wx)
    R = c * eye + s * wx + (1.0 - c) * (w[..., :, None] * w[..., None, :])
    R = torch.where((theta > 0)[..., None], R, eye)
    return torch.cat([R, t[..., None]], dim=-1)


def _p3p_init(points_3d, points_2d, camera_matrix, order_key):
    """The reference's initialisation (un_pnp_utils.py:25-31): OpenCV P3P on the four points with the largest key."""
    import cv2
    try:
        dist_coeffs = uncertainty_pnp.dist_coeffs
    except AttributeError:
        dist_coeffs = np.zeros(shape=[8, 1], dtype=np.float64)
    idxs = np.argsort(order_key)[-4:]
    _, r_exp, t = cv2.solvePnP(np.expand_dims(points_3d[idxs, :], 0), np.expand_dims(points_2d[idxs, :], 0),
                               camera_matrix, dist_coeffs, None, None, False, flags=cv2.SOLVEPNP_P3P)
    return r_exp, t


def _solve_one(points_2d, weights_2d, points_3d, camera_matrix, order_key, init_rt, device):
    pn = points_2d.shape[0]
    assert points_3d.shape[0] == pn and pn >= 4
    points_3d = points_3d.astype(np.float64)
    points_2d = points_2d.astype(np.float64)
    weights_2d = weights_2d.astype(np.float64)
    camera_matrix = camera_matrix.astype(np.float64)
    if init_rt is None:
        r_exp, t = _p3p_init(points_3d, points_2d, camera_matrix, order_key)
        init_rt = np.concatenate([r_exp, t], 0).reshape(6)
    init_rt = np.asarray(init_rt, np.float64).reshape(6)
    dev = torch.device(device)
    if pn == 4:                                           # no other points (un_pnp_utils.py:33-37)
        return rodrigues(torch.from_numpy(init_rt)[None])[0].numpy()
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    rt = uncertainty_pnp_batch(tt(points_2d)[None], tt(weights_2d)[None], tt(points_3d), tt(camera_matrix), tt(init_rt)[None])
    return rodrigues(rt)[0].cpu().numpy()


def uncertainty_pnp(points_2d, weights_2d, points_3d, camera_matrix, init_rt=None, device="cuda"):
    """Twin of un_pnp_utils.uncertainty_pnp (:6-57): numpy in, 3x4 [R|t] out.
    points_2d [pn,2], weights_2d [pn,3] (wxx,wxy,wyy), points_3d [pn,3], camera_matrix [3,3]."""
    weights_2d = np.asarray(weights_2d)
    return _solve_one(np.asarray(points_2d), weights_2d, np.asarray(points_3d), np.asarray(camera_matrix),
                      weights_2d[:, 0].astype(np.float64) + weights_2d[:, 1].astype(np.float64), init_rt, device)


def uncertainty_pnp_v2(points_2d, covars, points_3d, camera_matrix, type="single", init_rt=None, device="cuda"):
    """Twin of un_pnp_utils.uncertainty_pnp_v2 (:60-121): isotropic weights 1/lambda_max(cov), 0 where cov[0,0] < 1e-5."""
    covars = np.asarray(covars)
    pn = np.asarray(points_2d).shape[0]
    assert covars.shape[0] == pn
    w = []
    for pi in range(pn):
        if covars[pi, 0, 0] < 1e-5:
            w.append(0.0)
        else:
            w.append(1.0 / np.max(np.linalg.eigvals(covars[pi])))
    w = np.asarray(w, np.float64)
    weights_2d = np.stack([w, np.zeros(pn), w], 1)
    return _solve_one(np.asarray(points_2d), weights_2d, np.asarray(points_3d), np.asarray(camera_matrix), w, init_rt, device)
