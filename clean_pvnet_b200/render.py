"""T-LESS's VSD on the device, without OpenGL (DESIGN.md section 8f; the kernels are csrc/render.cu):

    render_depth_batch(pts, faces, poses, K, size)         what DepthRender.render (lib/utils/renderer/opengl_utils.py:
                                                           405-490) renders, for n poses -> float32 [n,H,W] CUDA tensor
    vsd_batch(pts, faces, pose_est, pose_gt, K, depth_test, pairs)
                                                           vsd_utils.vsd with T-LESS's 'step' cost for n (estimate, ground
                                                           truth, image) rows, as Evaluator.vsd_metric calls it -> float64 [n]
    install_depth_renderer_as_reference()                  `lib.utils.renderer.opengl_utils` and `lib.utils.vsd.renderer`
                                                           bind this module: DepthRender / render(mode='depth') without glumpy

and T-LESS's instance masks (DESIGN.md section 8k), what lib/datasets/tless/handle_test_data.py:get_mask builds with OpenGL:

    instance_masks_batch(meshes, mesh_index, obj_ids, image_index, poses, K, size)
                                                           label map, unoccluded and visible pixel counts and bounding box
                                                           of every instance of B images -> CUDA tensors
    instance_masks_from_depth(depth, slot, obj_ids, image_index)
                                                           the same from given depth images (the compose step alone)
    install_tless_renderer_as_reference()                  `lib.datasets.tless.opengl_backend` binds this module

Poses are [R|t] in the units of the mesh: the evaluator renders its model in millimetres with t * 1000.  Nothing is
copied to the host and nothing waits for the device; every chunk is planned from the shapes.
"""
import ctypes
import sys

import numpy as np
import torch

from . import _lib
from .nn import _call, _workspace

# T-LESS's settings (lib/utils/tless/tless_config.py: vsd_delta, vsd_tau, error_thresh_vsd) and the evaluator's clip planes
VSD_DELTA, VSD_TAU, VSD_THRESHOLD = 15, 20, 0.3
CLIP_NEAR, CLIP_FAR = 100, 10000
_MAX_QUEUE = 1 << 26            # render queue entries (4 bytes each) per launch: the poses of a launch times the faces


def _device(*ts):
    for t in ts:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _mesh(pts, faces):
    """(pts, faces) as tensors, shape-checked where they are (nothing moves before every argument is checked)."""
    p, f = torch.as_tensor(pts), torch.as_tensor(faces)
    if p.dim() != 2 or p.shape[1] != 3:
        raise RuntimeError(f"pts must be [V,3], got {list(p.shape)}")
    if f.dim() != 2 or f.shape[1] != 3:
        raise RuntimeError(f"faces must be [F,3], got {list(f.shape)}")
    return p, f


def _to(t, dev, dtype):
    return t.to(device=dev, dtype=dtype).contiguous()


def _size(size):
    W, H = (int(s) for s in size)
    if W < 0 or H < 0:
        raise RuntimeError(f"size must be (width, height) >= 0, got {size}")
    return W, H


def _render(p, f, poses, K, k_stride, W, H, near, far, out):
    """pvb_render_depth over the poses in launches whose queue stays within _MAX_QUEUE entries."""
    n, F = int(poses.shape[0]), int(f.shape[0])
    step = max(1, min(65535, _MAX_QUEUE // max(F, 1)))
    dev = poses.device
    for s in range(0, n, step):
        m = min(step, n - s)
        nbytes = _lib.load().pvb_render_depth_workspace_bytes(m, F)
        _call("pvb_render_depth", dev, p, int(p.shape[0]), f, F, poses[s:s + m], m, K[s:s + m] if k_stride else K,
              k_stride, out[s:s + m], H, W, float(near), float(far), _workspace(nbytes, dev), nbytes)
    return out


def render_depth_batch(pts, faces, poses, K, size, near=CLIP_NEAR, far=CLIP_FAR):
    """The depth image DepthRender.render(size, near, far, K, R, t) returns (lib/utils/renderer/opengl_utils.py:405-490),
    for n poses at once: pts [V,3] (rounded to float32, as the vertex buffer is), faces [F,3], poses [n,3,4] ([R|t],
    rounded to float32 like the shader's view matrix), K [3,3] or [n,3,3], size (width, height) like the reference's
    im_size.  Pixel (r, c) holds the camera-frame Z of the nearest surface along the ray through (c + 0.5, r + 0.5) with
    near <= Z <= far, else 0.  Returns float32 [n,H,W] on the device of poses (the current CUDA device when it is not a
    CUDA tensor); bit-identical run to run, and each pose's image independent of the batch."""
    p, f = _mesh(pts, faces)
    pz, km = torch.as_tensor(poses), torch.as_tensor(K)
    if pz.dim() != 3 or tuple(pz.shape[1:]) != (3, 4):
        raise RuntimeError(f"poses must be [n,3,4], got {list(pz.shape)}")
    n = int(pz.shape[0])
    if tuple(km.shape) not in ((3, 3), (n, 3, 3)):
        raise RuntimeError(f"K must be [3,3] or [{n},3,3], got {list(km.shape)}")
    W, H = _size(size)
    if not (0 < float(near) <= float(far) < float("inf")):
        raise RuntimeError(f"need 0 < near <= far < inf, got {near}, {far}")
    dev = _device(pz, p)
    out = torch.empty((n, H, W), dtype=torch.float32, device=dev)
    return _render(_to(p, dev, torch.float32), _to(f, dev, torch.int32), _to(pz, dev, torch.float64),
                   _to(km, dev, torch.float64), 0 if km.dim() == 2 else 9, W, H, near, far, out)


def vsd_batch(pts, faces, pose_est, pose_gt, K, depth_test, pairs, delta=VSD_DELTA, tau=VSD_TAU, near=CLIP_NEAR,
              far=CLIP_FAR, max_render_bytes=1 << 30):
    """vsd_utils.vsd (lib/utils/vsd/vsd_utils.py:5-48) with the 'step' cost, on the distance images and visibility masks
    Evaluator.vsd_metric (lib/evaluators/tless_test/pvnet.py:66-105) builds for it, for n rows at once.
        pts, faces   the mesh (the evaluator's model: millimetres)
        pose_est     [n_e,3,4] estimated poses, pose_gt [n_g,3,4] ground-truth poses, in the mesh's units (t * 1000)
        K            [3,3] shared, or [B,3,3] per image (each pose is rendered with the K of the image its rows name)
        depth_test   [B,H,W] test depth images (the evaluator's inout.load_depth(path) * 0.1), rounded to float32
        pairs        [n,3] integer rows (estimate index, ground-truth index, image index)
    Each pose is rendered once (at near / far) when all of them fit in max_render_bytes, else in windows of that size.
    Returns float64 [n] on the device of depth_test: e, exactly the reference's for the same rendered depth; a row with an
    index out of range gives NaN.  Evaluator.vsd_metric's flag of image b is any(e[i] < 0.3 for the rows of b)."""
    p, f = _mesh(pts, faces)
    dt, pe, pg, km, pr = (torch.as_tensor(t) for t in (depth_test, pose_est, pose_gt, K, pairs))
    if dt.dim() != 3:
        raise RuntimeError(f"depth_test must be [B,H,W], got {list(dt.shape)}")
    B, H, W = (int(s) for s in dt.shape)
    for name, t in (("pose_est", pe), ("pose_gt", pg)):
        if t.dim() != 3 or tuple(t.shape[1:]) != (3, 4):
            raise RuntimeError(f"{name} must be [n,3,4], got {list(t.shape)}")
    if tuple(km.shape) not in ((3, 3), (B, 3, 3)):
        raise RuntimeError(f"K must be [3,3] or [{B},3,3], got {list(km.shape)}")
    if pr.dim() != 2 or pr.shape[1] != 3 or pr.dtype.is_floating_point or pr.dtype == torch.bool:
        raise RuntimeError(f"pairs must be an integer [n,3] tensor, got {pr.dtype} {list(pr.shape)}")
    if not (0 < float(near) <= float(far) < float("inf")):
        raise RuntimeError(f"need 0 < near <= far < inf, got {near}, {far}")
    dev = _device(dt, pe, pg, pr)
    p, f, dt = _to(p, dev, torch.float32), _to(f, dev, torch.int32), _to(dt, dev, torch.float32)
    pe, pg, km, pr = _to(pe, dev, torch.float64), _to(pg, dev, torch.float64), _to(km, dev, torch.float64), \
        _to(pr, dev, torch.int32)
    n, ne, ng = int(pr.shape[0]), int(pe.shape[0]), int(pg.shape[0])
    e = torch.full((n,), float("nan"), dtype=torch.float64, device=dev)
    if n == 0 or ne == 0 or ng == 0 or B == 0:
        return e

    def pose_k(count, col):
        """The K of each pose: the K of the image of (one of) its rows; clamped indices keep the gather in range."""
        if km.dim() == 2:
            return km, 0
        img = torch.zeros(count, dtype=torch.int64, device=dev)
        img.scatter_(0, pr[:, col].long().clamp(0, count - 1), pr[:, 2].long().clamp(0, B - 1))
        return km[img].contiguous(), 9

    ke, kes = pose_k(ne, 0)
    kg, kgs = pose_k(ng, 1)
    per = max(H * W * 4, 1)
    if (ne + ng) * per <= max_render_bytes:
        we, wg = ne, ng
    else:
        we = wg = max(1, max_render_bytes // 2 // per)
    nbytes = _lib.load().pvb_vsd_workspace_bytes(n)
    ws = _workspace(nbytes, dev)
    kimg = 0 if km.dim() == 2 else 9
    est_buf = torch.empty((min(we, ne), H, W), dtype=torch.float32, device=dev)
    gt_buf = torch.empty((min(wg, ng), H, W), dtype=torch.float32, device=dev)
    gt_done = None
    for e0 in range(0, ne, we):
        me = min(we, ne - e0)
        _render(p, f, pe[e0:e0 + me], ke[e0:e0 + me] if kes else ke, kes, W, H, near, far, est_buf[:me])
        for g0 in range(0, ng, wg):
            mg = min(wg, ng - g0)
            if gt_done != g0:                                # one window of ground truths stays rendered across estimates
                _render(p, f, pg[g0:g0 + mg], kg[g0:g0 + mg] if kgs else kg, kgs, W, H, near, far, gt_buf[:mg])
                gt_done = g0
            _call("pvb_vsd", dev, dt, B, est_buf, me, e0, gt_buf, mg, g0, pr, n, km, kimg, H, W, float(delta),
                  float(tau), e, ws, nbytes)
    return e


# ---- T-LESS's instance masks (DESIGN.md section 8k) ------------------------------------------------------------------

def _host_ints(x, name):
    """A host table (from gt.yml) as a 1-D int64 numpy array; a CUDA tensor is refused rather than copied back."""
    if isinstance(x, torch.Tensor) and x.is_cuda:
        raise RuntimeError(f"{name} must be host data (a list, numpy array or CPU tensor), got a CUDA tensor")
    a = np.asarray(x.numpy() if isinstance(x, torch.Tensor) else x)
    if a.ndim != 1 or not (a.size == 0 or np.issubdtype(a.dtype, np.integer)):
        raise RuntimeError(f"{name} must be a 1-D integer table, got {a.dtype} {list(a.shape)}")
    return a.astype(np.int64)


def _upload(a, dev):
    """A host index table on the device without waiting for it: pinned staging and a non-blocking copy."""
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)


def _instance_plan(obj_ids, image_index, B):
    """Checks the tables and returns image_first [B+1] (image b's instances are [first[b], first[b+1]))."""
    n = len(image_index)
    if len(obj_ids) != n:
        raise RuntimeError(f"obj_ids and image_index must have one entry per instance, got {len(obj_ids)} and {n}")
    if n and (np.any(np.diff(image_index) < 0) or image_index[0] < 0 or image_index[-1] >= B):
        raise RuntimeError(f"image_index must be non-decreasing (each image's instances together, in gt order) and in "
                           f"[0, {B})")
    first = np.searchsorted(image_index, np.arange(B + 1), side="left")
    rank = np.arange(n) - first[image_index] if n else np.zeros(0, np.int64)
    label = obj_ids * 1000 + rank
    if n and (label.min() < -32768 or label.max() > 32767):
        raise RuntimeError("obj_id * 1000 + instance_id must fit int16 (the label map's type)")
    return first


def _compose(depth, n_depth, slot, obj, first, b0, b1, H, W, label, a_num, p_num, bbox, dev):
    """pvb_instance_masks over images [b0, b1), split where an image has no instance (its label map stays 0)."""
    slot32, obj32 = np.ascontiguousarray(slot, np.int32), np.ascontiguousarray(obj, np.int32)
    b = b0
    while b < b1:
        if first[b] == first[b + 1]:
            b += 1
            continue
        e = b
        while e < b1 and e - b < 65535 and first[e] != first[e + 1]:
            e += 1
        f32 = np.ascontiguousarray(first[b:e + 1], np.int32)
        nbytes = _lib.load().pvb_instance_masks_workspace_bytes(e - b, int(f32[-1] - f32[0]))
        _call("pvb_instance_masks", dev, depth, n_depth, slot32.ctypes.data_as(ctypes.c_void_p),
              obj32.ctypes.data_as(ctypes.c_void_p), len(obj32), f32.ctypes.data_as(ctypes.c_void_p), e - b, H, W,
              label[b], a_num, p_num, bbox, _workspace(nbytes, dev), nbytes)
        b = e


def _mask_outputs(B, n, H, W, first, dev):
    empty = bool(np.any(first[1:] == first[:-1]))
    label = (torch.zeros if empty else torch.empty)((B, H, W), dtype=torch.int16, device=dev)
    return (label, torch.empty(n, dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.int64, device=dev),
            torch.empty((n, 4), dtype=torch.int32, device=dev))


def instance_masks_from_depth(depth, slot, obj_ids, image_index):
    """handle_test_data.get_mask's compose step (lib/datasets/tless/handle_test_data.py:81-134) on given depth images:
        depth        [S,H,W] depth slots in mm, as pvb_render_depth writes them (rounded to float32)
        slot         host [n]: instance i reads depth[slot[i]]
        obj_ids      host [n]: each instance's obj_id
        image_index  host [n], non-decreasing: each instance's image; instance_id is its rank within the image
    Each image b in [0, max(image_index)] composes its instances in order, as update_mask does on
    opengl_renderer.render's depth / 1000.  Returns (label int16 [B,H,W], a_pixel_num int64 [n], pixel_num int64 [n],
    bbox int32 [n,4]) on the device of depth: the mask/*.png label map (obj_id * 1000 + instance_id), pixel_num.pkl's
    count of each instance's rendered pixels, the count of its labelled pixels, and cv2.boundingRect (x, y, w, h) of those
    ((0, 0, 0, 0) when it has none).  Exact integers, bit-identical run to run; an image's outputs depend on nothing else."""
    d = torch.as_tensor(depth)
    if d.dim() != 3:
        raise RuntimeError(f"depth must be [S,H,W], got {list(d.shape)}")
    S, H, W = (int(s) for s in d.shape)
    sl, obj, img = _host_ints(slot, "slot"), _host_ints(obj_ids, "obj_ids"), _host_ints(image_index, "image_index")
    if len(sl) != len(img):
        raise RuntimeError(f"slot and image_index must have one entry per instance, got {len(sl)} and {len(img)}")
    if len(sl) and (sl.min() < 0 or sl.max() >= S):
        raise RuntimeError(f"slot must index depth's {S} images")
    n = len(img)
    B = int(img[-1]) + 1 if n else 0
    first = _instance_plan(obj, img, B)
    dev = _device(d)
    d = _to(d, dev, torch.float32)
    out = _mask_outputs(B, n, H, W, first, dev)
    _compose(d, S, sl, obj, first, 0, B, H, W, *out, dev)
    return out


def instance_masks_batch(meshes, mesh_index, obj_ids, image_index, poses, K, size, near=10, far=10000,
                         max_render_bytes=1 << 30):
    """handle_test_data.get_mask (lib/datasets/tless/handle_test_data.py:93-134) for B images at once, without OpenGL:
        meshes       list of (pts [V,3], faces [F,3]) in mm (the CAD models as load_ply returns them)
        mesh_index   host [n]: the mesh of each instance; obj_ids host [n]: its obj_id (gt.yml's obj_id)
        image_index  host [n], non-decreasing: its image (instance_id is its rank within the image, gt_'s order)
        poses        [n,3,4] [R|t] with t in mm (cam_t_m2c, as opengl_renderer.render passes t * 1000)
        K            [3,3] shared or [B,3,3] per image; size (width, height)
    Each instance is rendered as opengl_renderer.render renders it (pvb_render_depth at clip planes near / far) into a
    slot of a scratch window that holds whole images within max_render_bytes, then the window's images are composed as
    instance_masks_from_depth does.  B is K's first dimension, else max(image_index) + 1.  Returns (label int16 [B,H,W],
    a_pixel_num int64 [n], pixel_num int64 [n], bbox int32 [n,4]) on the device of poses (the current CUDA device when
    it is not a CUDA tensor).  Nothing is copied back to the host; with the meshes, poses and K on the device nothing
    waits for it either (the host tables go up through pinned, non-blocking copies)."""
    mi, obj, img = _host_ints(mesh_index, "mesh_index"), _host_ints(obj_ids, "obj_ids"), _host_ints(image_index,
                                                                                                    "image_index")
    ms = [_mesh(p, f) for p, f in meshes]
    pz, km = torch.as_tensor(poses), torch.as_tensor(K)
    n = len(img)
    if pz.dim() != 3 or tuple(pz.shape) != (n, 3, 4):
        raise RuntimeError(f"poses must be [{n},3,4], got {list(pz.shape)}")
    if len(mi) != n:
        raise RuntimeError(f"mesh_index must have one entry per instance, got {len(mi)} for {n}")
    if n and (mi.min() < 0 or mi.max() >= len(ms)):
        raise RuntimeError(f"mesh_index must index the {len(ms)} meshes")
    if km.dim() == 3 and tuple(km.shape[1:]) == (3, 3):
        B = int(km.shape[0])
    elif tuple(km.shape) == (3, 3):
        B = int(img[-1]) + 1 if n else 0
    else:
        raise RuntimeError(f"K must be [3,3] or [B,3,3], got {list(km.shape)}")
    W, H = _size(size)
    if not (0 < float(near) <= float(far) < float("inf")):
        raise RuntimeError(f"need 0 < near <= far < inf, got {near}, {far}")
    first = _instance_plan(obj, img, B)
    dev = _device(pz, km, *(t for m in ms for t in m))
    out = _mask_outputs(B, n, H, W, first, dev)
    if n == 0 or H * W == 0:
        if n:
            _compose(None, 1, np.zeros(n, np.int64), obj, first, 0, B, H, W, *out, dev)
        return out
    # windows of whole images within max_render_bytes (at least one image each)
    per = H * W * 4
    windows, b0 = [], 0
    while b0 < B:
        b1 = b0 + 1
        while b1 < B and (first[b1 + 1] - first[b0]) * per <= max_render_bytes:
            b1 += 1
        windows.append((b0, b1))
        b0 = b1
    # within a window the instances are rendered mesh by mesh: order = window-major, then mesh, then instance
    order = np.concatenate([first[w0] + np.argsort(mi[first[w0]:first[w1]], kind="stable") for w0, w1 in windows])
    pos = np.empty(n, np.int64)
    pos[order] = np.arange(n)
    identity = bool(np.all(order == np.arange(n)))
    perm = None if identity else _upload(order, dev)
    pz = _to(pz, dev, torch.float64)
    pz = pz if identity else pz.index_select(0, perm)
    km = _to(km, dev, torch.float64)
    if km.dim() == 3:
        kimg = _upload(img[order], dev)
        km, kst = km.index_select(0, kimg).contiguous(), 9
    else:
        kst = 0
    mesh_dev = {}
    width = max(int(first[w1] - first[w0]) for w0, w1 in windows)
    buf = torch.empty((width, H, W), dtype=torch.float32, device=dev)
    for w0, w1 in windows:
        s0, s1 = int(first[w0]), int(first[w1])
        if s0 == s1:
            continue                                   # images without instances: their label maps are zero-filled
        sorted_mesh = mi[order[s0:s1]]
        starts = np.flatnonzero(np.r_[True, sorted_mesh[1:] != sorted_mesh[:-1]])
        for a, z in zip(starts, np.r_[starts[1:], s1 - s0]):
            k = int(sorted_mesh[a])
            if k not in mesh_dev:
                mesh_dev[k] = (_to(ms[k][0], dev, torch.float32), _to(ms[k][1], dev, torch.int32))
            p, f = mesh_dev[k]
            _render(p, f, pz[s0 + a:s0 + z], km[s0 + a:s0 + z] if kst else km, kst, W, H, near, far, buf[a:z])
        _compose(buf, s1 - s0, pos - s0, obj, first, w0, w1, H, W, *out, dev)
    return out


# ---- drop-in twins of the reference's OpenGL renderers (depth only) --------------------------------------------------

def _pose(R, t):
    return np.hstack([np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3, 1)])[None]


class DepthRender:
    """Twin of lib/utils/renderer/opengl_utils.py:405-490 (and lib/utils/vsd/renderer.py's DepthRender) on the CUDA
    renderer: no window, no GL context.  render(im_size, clip_near, clip_far, K, R, t) returns the reference's numpy
    float32 [h,w] depth image."""

    def __init__(self, model, im_size, texture=None, bg_color=(0.0, 0.0, 0.0, 0.0), ambient_weight=0.5, shading='flat',
                 mode='rgb+depth'):
        dev = torch.device("cuda", torch.cuda.current_device())
        self.im_size = im_size
        p, f = _mesh(np.asarray(model['pts'], np.float32), np.asarray(model['faces']).astype(np.int32))
        self._pts, self._faces = _to(p, dev, torch.float32), _to(f, dev, torch.int32)

    def render(self, im_size, clip_near, clip_far, K, R, t):
        return render_depth_batch(self._pts, self._faces, _pose(R, t), np.asarray(K, np.float64), im_size, clip_near,
                                  clip_far)[0].cpu().numpy()


class NormalRender:
    """opengl_utils.NormalRender renders normals, which this project does not render."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("only depth is rendered without OpenGL (NormalRender is not available)")


def render(model, im_size, K, R, t, clip_near=100, clip_far=2000, texture=None, surf_color=None,
           bg_color=(0.0, 0.0, 0.0, 0.0), ambient_weight=0.5, shading='flat', mode='rgb+depth'):
    """Twin of opengl_utils.render / lib/utils/vsd/renderer.py's render for mode='depth' (the only mode VSD uses): the
    numpy float32 [h,w] depth image.  Every other mode raises NotImplementedError."""
    if mode != 'depth':
        raise NotImplementedError(f"only mode='depth' is rendered without OpenGL (got mode={mode!r})")
    assert {'pts', 'faces'}.issubset(set(model.keys()))
    return DepthRender(model, im_size).render(im_size, clip_near, clip_far, K, R, t)


def install_depth_renderer_as_reference():
    """Makes `from lib.utils.renderer import opengl_utils` (lib/utils/icp/icp_utils.py:1) and `from . import renderer` in
    lib/utils/vsd/vsd_utils.py:2 bind this module, so vsd_utils, icp_utils and the T-LESS evaluator's vsd_metric import
    and run without glumpy or a GL context.  Only the two leaf modules are replaced; `lib`, `lib.utils`, ... stay the real
    packages whenever they exist.  Idempotent."""
    from ._dropin import reference_package
    this = sys.modules[__name__]
    for parent_name, leaf in (("lib.utils.renderer", "opengl_utils"), ("lib.utils.vsd", "renderer")):
        parent = reference_package(parent_name)
        sys.modules[f"{parent_name}.{leaf}"] = this
        setattr(parent, leaf, this)
    return this


def install_tless_renderer_as_reference():
    """Makes `from lib.datasets.tless import opengl_backend` (lib/datasets/tless/opengl_renderer.py:3) bind this module,
    so opengl_renderer, handle_test_data and handle_ag_data import without glumpy, and opengl_renderer.render(model, pose,
    K, w, h) returns this renderer's depth / 1000 (its render(..., clip_near=10, clip_far=10000, mode='depth')).  Only
    the leaf module is replaced; `lib.datasets.tless` stays the real package whenever it exists.  Idempotent."""
    from ._dropin import reference_package
    this = sys.modules[__name__]
    parent = reference_package("lib.datasets.tless")
    sys.modules["lib.datasets.tless.opengl_backend"] = this
    setattr(parent, "opengl_backend", this)
    return this
