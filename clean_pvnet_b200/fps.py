"""Twin of clean-pvnet's `lib/csrc/fps` (the cffi extension tools/handle_custom_dataset.py imports to pick a custom object's
keypoints) on the device kernel of csrc/fps.cu.

    farthest_point_sampling(pts, sn, init_center=False)   fps_utils.py:5-21: numpy [pn,3] in, float32 pts[idxs] [sn,3] out
    farthest_point_sampling_batch(points, sn, init_center=True, counts=None, starts=None)
                                                          B clouds in one launch: CUDA [B,N,3] -> int32 [B,sn]
    install_fps_as_reference_module()                     `from lib.csrc.fps import fps_utils` binds this module

The indices are the reference's element for element (pvb_farthest_point_sampling in include/pvnet_vote_b200.h); there is
no CPU implementation behind them.  One deviation: the reference's random start is `rand() % pn` after `srand(time(0))`,
which cannot be reproduced; here it is `np.random.randint(pn)`, so a run repeats under `np.random.seed`.
"""
import ctypes
import sys

import numpy as np
import torch

from . import _lib


def _host_i32(v, b, name):
    a = np.ascontiguousarray(torch.as_tensor(v).cpu().numpy() if isinstance(v, torch.Tensor) else v, dtype=np.int64)
    if a.shape != (b,):
        raise RuntimeError(f"{name} must have one entry per cloud ({b}), got shape {list(a.shape)}")
    if a.size and (a.min() < -2 ** 31 or a.max() >= 2 ** 31):
        raise RuntimeError(f"{name} must fit int32")
    return a.astype(np.int32)


def farthest_point_sampling_batch(points, sn, init_center=True, counts=None, starts=None):
    """Farthest-point sampling of B clouds in one launch, with the reference's arithmetic and tie rule.  points is a CUDA
    tensor [B,N,3] (converted to contiguous float32); cloud b is its first counts[b] rows (all N when counts is None).
    init_center: start from the point farthest from the centre of the cloud's bounding box
    (farthest_point_sampling_init_center); otherwise cloud b starts at starts[b], drawn with np.random.randint(counts[b])
    in cloud order when starts is None.  counts and starts are host sequences (a CUDA tensor is copied to the host).
    Returns int32 [B,sn] on points' device; the call does not wait for the device."""
    if not (isinstance(points, torch.Tensor) and points.is_cuda):
        raise RuntimeError("points must be a CUDA tensor")
    if points.dim() != 3 or points.shape[2] != 3:
        raise RuntimeError(f"points must be [B,N,3], got {list(points.shape)}")
    sn = int(sn)
    if sn < 0:
        raise RuntimeError(f"sn must be >= 0, got {sn}")
    b, n = int(points.shape[0]), int(points.shape[1])
    cnt = np.full(b, n, np.int32) if counts is None else _host_i32(counts, b, "counts")
    if init_center:
        st = None
    elif starts is None:
        st = np.array([np.random.randint(int(c)) if c > 0 else 0 for c in cnt], np.int32)
    else:
        st = _host_i32(starts, b, "starts")
    dev = points.device
    p = points.float().contiguous()
    idxs = torch.empty((b, sn), dtype=torch.int32, device=dev)
    lib = _lib.load()
    nbytes = lib.pvb_fps_workspace_bytes(b, n)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes else None
    with torch.cuda.device(dev):
        _lib.check(lib.pvb_farthest_point_sampling(
            ctypes.c_void_p(p.data_ptr()), cnt.ctypes.data, None if st is None else st.ctypes.data,
            int(bool(init_center)), ctypes.c_void_p(idxs.data_ptr()), b, n, sn,
            None if ws is None else ctypes.c_void_p(ws.data_ptr()), nbytes,
            ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return idxs


def farthest_point_sampling(pts, sn, init_center=False):
    """fps_utils.farthest_point_sampling (lib/csrc/fps/fps_utils.py:5-21): pts [pn,3] (rounded to float32 like the
    reference) -> float32 pts[idxs] [sn,3], the sn farthest-point samples.  init_center=False starts at
    np.random.randint(pn) (the reference: rand() % pn after srand(time(0))).  Runs on the current CUDA device."""
    pn, _ = pts.shape
    assert (pts.shape[1] == 3)
    pts = np.ascontiguousarray(pts, np.float32)
    dev = torch.device("cuda", torch.cuda.current_device())
    idxs = farthest_point_sampling_batch(torch.from_numpy(pts[None]).to(dev), sn, init_center=init_center)
    return pts[idxs.cpu().numpy()[0]]


def install_fps_as_reference_module():
    """Makes `from lib.csrc.fps import fps_utils` (tools/handle_custom_dataset.py:4) bind this module, so custom-object
    preparation runs without the cffi extension `lib.csrc.fps._ext` ever being built or imported.  Only the leaf
    `lib.csrc.fps.fps_utils` is replaced; `lib`, `lib.csrc` and `lib.csrc.fps` stay the real packages whenever they exist
    (see install_nn_as_reference_module).  Idempotent."""
    from ._dropin import reference_package
    this = sys.modules[__name__]
    parent = reference_package("lib.csrc.fps")
    sys.modules["lib.csrc.fps.fps_utils"] = this
    parent.fps_utils = this
    return this
