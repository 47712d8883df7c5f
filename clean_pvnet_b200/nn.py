"""Twin of clean-pvnet's `lib/csrc/nn` (the cffi extension both evaluators import, lib/evaluators/linemod/pvnet.py:20 and
tless_test/pvnet.py:13) on the device kernels of csrc/nn.cu, plus the evaluators' ADD / ADD-S distance for a whole batch.

    find_nearest_point_idx(ref_pts, que_pts)              nn_utils.py:5-20: numpy in, numpy int32 [pn2] out
    nearest_point_idx(ref, que, exclude_self=False)       batched CUDA tensors [b,pn1,dim], [b,pn2,dim] -> int32 [b,pn2]
    add_metric_batch(model, pose_pred, pose_gt, syn)      mean_dist of Evaluator.add_metric (linemod/pvnet.py:68-82) for
                                                          n pose pairs -> float64 [n] CUDA tensor
    install_nn_as_reference_module()                      `from lib.csrc.nn import nn_utils` binds this module

The indices are the reference kernel's bit for bit (pvb_nearest_point_idx in include/pvnet_vote_b200.h); there is no CPU
implementation behind them.
"""
import ctypes
import sys

import numpy as np
import torch

from . import _lib


def _call(entry, dev, *args):
    """lib.<entry>(*args, stream) on the current stream of `dev`; tensors go in as their device pointers, None as NULL."""
    lib = _lib.load()
    args = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        _lib.check(getattr(lib, entry)(*args, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))


def _workspace(nbytes, dev):
    return torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None


def nearest_point_idx(ref, que, exclude_self=False):
    """For every query point que[i][q], the index of its nearest reference point in ref[i] (the first one in index order
    among equal distances), with the reference kernel's fp32 arithmetic.  ref [b,pn1,dim] and que [b,pn2,dim] are CUDA
    tensors on one device (converted to contiguous float32), dim 2 or 3.  exclude_self: reference point q is not a
    candidate for query q (the reference's `exclude_self`).  Returns int32 [b,pn2] on that device; no host sync."""
    if not (isinstance(ref, torch.Tensor) and isinstance(que, torch.Tensor) and ref.is_cuda and que.is_cuda):
        raise RuntimeError("ref and que must be CUDA tensors")
    if ref.device != que.device:
        raise RuntimeError(f"ref and que must be on one device, got {ref.device} and {que.device}")
    if ref.dim() != 3 or que.dim() != 3 or ref.shape[0] != que.shape[0] or ref.shape[2] != que.shape[2]:
        raise RuntimeError(f"ref must be [b,pn1,dim] and que [b,pn2,dim], got {list(ref.shape)} and {list(que.shape)}")
    b, pn1, dim = (int(s) for s in ref.shape)
    pn2 = int(que.shape[1])
    if dim not in (2, 3):
        raise RuntimeError(f"dim must be 2 or 3, got {dim}")
    dev = ref.device
    r, q = ref.float().contiguous(), que.float().contiguous()
    idxs = torch.empty((b, pn2), dtype=torch.int32, device=dev)
    nbytes = _lib.load().pvb_nearest_point_workspace_bytes(b, pn1, pn2)
    ws = _workspace(nbytes, dev)
    _call("pvb_nearest_point_idx", dev, r, q, idxs, b, pn1, pn2, dim, int(bool(exclude_self)), ws, nbytes)
    return idxs


def find_nearest_point_idx(ref_pts, que_pts):
    """nn_utils.find_nearest_point_idx (lib/csrc/nn/nn_utils.py:5-20): ref_pts [pn1,dim], que_pts [pn2,dim] numpy arrays
    (rounded to float32 like the reference), dim 2 or 3 -> int32 [pn2], the index of each query's nearest reference point.
    Runs on the current CUDA device."""
    assert (ref_pts.shape[1] == que_pts.shape[1] and 1 < que_pts.shape[1] <= 3)
    dev = torch.device("cuda", torch.cuda.current_device())
    ref = torch.from_numpy(np.ascontiguousarray(ref_pts[None, :, :], np.float32)).to(dev)
    que = torch.from_numpy(np.ascontiguousarray(que_pts[None, :, :], np.float32)).to(dev)
    return nearest_point_idx(ref, que).cpu().numpy()[0]


def add_metric_batch(model, pose_pred, pose_gt, syn):
    """The mean distance of Evaluator.add_metric (lib/evaluators/linemod/pvnet.py:68-82) for n pose pairs at once:
    model [pn,3] (shared), pose_pred / pose_gt [n,3,4] ([R|t]); tensors or arrays, computed in float64.
    syn=False (ADD): mean |pred_i - target_i|; syn=True (ADD-S): every target point to its nearest predicted point, found
    on both clouds rounded to float32 exactly like nn_utils + the reference kernel.  Returns float64 [n] on the device of
    pose_pred (the current CUDA device when it is not a CUDA tensor); compare with 0.1 * diameter yourself.
    T-LESS's adi_metric (tless_test/pvnet.py:107-117) is this over every (prediction, ground truth) pair."""
    dev = pose_pred.device if isinstance(pose_pred, torch.Tensor) and pose_pred.is_cuda else \
        torch.device("cuda", torch.cuda.current_device())
    f64 = lambda t: torch.as_tensor(t).to(device=dev, dtype=torch.float64).contiguous()   # noqa: E731
    m, pp, pg = f64(model), f64(pose_pred), f64(pose_gt)
    if m.dim() != 2 or m.shape[1] != 3:
        raise RuntimeError(f"model must be [pn,3], got {list(m.shape)}")
    if pp.dim() != 3 or tuple(pp.shape[1:]) != (3, 4) or pp.shape != pg.shape:
        raise RuntimeError(f"pose_pred and pose_gt must both be [n,3,4], got {list(pp.shape)} and {list(pg.shape)}")
    n, pn, s = int(pp.shape[0]), int(m.shape[0]), int(bool(syn))
    out = torch.empty(n, dtype=torch.float64, device=dev)
    nbytes = _lib.load().pvb_add_metric_workspace_bytes(n, pn, s)
    _call("pvb_add_metric", dev, m, pp, pg, out, n, pn, s, _workspace(nbytes, dev), nbytes)
    return out


def install_nn_as_reference_module():
    """Makes `from lib.csrc.nn import nn_utils` (lib/evaluators/linemod/pvnet.py:20, tless_test/pvnet.py:13) bind this
    module, so the evaluators import and run without the cffi extension `lib.csrc.nn._ext` ever being built or imported.
    Only the leaf `lib.csrc.nn.nn_utils` is replaced; `lib`, `lib.csrc` and `lib.csrc.nn` stay the real packages whenever
    they exist (see install_as_reference_module, which this complements).  Idempotent."""
    from ._dropin import reference_package
    this = sys.modules[__name__]
    parent = reference_package("lib.csrc.nn")
    sys.modules["lib.csrc.nn.nn_utils"] = this
    parent.nn_utils = this
    return this
