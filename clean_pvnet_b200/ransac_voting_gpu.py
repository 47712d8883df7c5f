"""Operator surface of the H100-native RANSAC voting layer.

Mirrors clean-pvnet's `lib/csrc/ransac_voting/ransac_voting_gpu.py` -- same function names,
positional/keyword signatures, return types -- so `lib/networks/pvnet/resnet18.py:5,71-75`
works unchanged (see INTEGRATION.md).  What differs is underneath: the per-image Python loop,
its ~50 launches and 5-6 host syncs per image, and the [hn,vn,tn] byte tensor are replaced by
a handful of batched sm_90a kernels behind one C-ABI call (csrc/*.cu), with no host sync.

Extra keyword-only arguments (all optional; the reference call sites never pass them):
    idxs       int32 [B,hn,K,2]  explicit sample pairs (the reference's per-image `idxs`, :145)
    selection  float [B,H,W]     explicit U(0,1) thinning draws (the reference's `selection`, :136)
    rng        "philox" (default): in-kernel counter-based sampling, no sync, result independent of
               batch sharding; seeded from torch's CPU generator (so torch.manual_seed applies)
               or `seed=`.
               "torch": consume torch's CUDA generator exactly like the reference does
               (uniform_ / random_ per image, in order), which makes results under
               torch.manual_seed(s) comparable with the reference bit-for-bit at the hypothesis
               level; costs the reference's per-image host syncs.
    img_base   global index of image 0 (multi-GPU shards keep one philox stream)
    capacity   per-image pixel capacity of the workspace (default max_num + 8*sqrt(max_num) + 64;
               H*W whenever selection is supplied)
    debug      also return the intermediates (tn, xy, dirs, hyp, counts, win; for v3 also normal_eq, the refit's
               float64 [B,K,5] normal equations (a00, a01, a11, b0, b1) summed over the winner's inliers)
"""
import math
import sys

import torch

from . import _lib
from . import ransac_voting as _ext

_MASK_DTYPES = {
    torch.uint8: _lib.PVB_MASK_U8, torch.bool: _lib.PVB_MASK_U8, torch.int8: _lib.PVB_MASK_I8,
    torch.int16: _lib.PVB_MASK_I16, torch.int32: _lib.PVB_MASK_I32, torch.int64: _lib.PVB_MASK_I64,
    torch.float32: _lib.PVB_MASK_F32, torch.float64: _lib.PVB_MASK_F64,
}

_workspaces = {}
_VALIDATE_CAPACITY = True      # tests switch it off to reach the device-side overflow report (PVB_ERR_CAPACITY)
RF_CHUNK = 2048                # pixels per refit CTA (RF_CHUNK in csrc/vote.cu): one partial of the normal equations each


def _workspace(device, nbytes):
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(int(nbytes * 1.25) + 256, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def _draw_seed():
    # CPU generator: no device sync, honours torch.manual_seed
    return int(torch.empty((), dtype=torch.int64).random_().item()) & 0xFFFFFFFFFFFFFFFF


def _check_inputs(mask, vertex):
    if not isinstance(mask, torch.Tensor) or not mask.is_cuda:
        raise RuntimeError("mask must be a CUDA tensor")
    if not isinstance(vertex, torch.Tensor) or not vertex.is_cuda:
        raise RuntimeError("vertex must be a CUDA tensor")
    if vertex.dim() != 5 or vertex.size(4) != 2:
        raise RuntimeError("vertex must be [b,h,w,vn,2]")
    if mask.dim() != 3 or tuple(mask.shape) != tuple(vertex.shape[:3]):
        raise RuntimeError("mask must be [b,h,w] matching vertex")
    if mask.device != vertex.device:
        raise RuntimeError("mask and vertex must be on the same device")
    if vertex.dtype != torch.float32:
        vertex = vertex.float()
    if mask.dtype in (torch.float16, torch.bfloat16):
        mask = mask.float()
    if mask.dtype not in _MASK_DTYPES:
        raise RuntimeError(f"unsupported mask dtype {mask.dtype}")
    return mask, vertex


_desc_cache = {}


def _cached_desc(lib, mask, vertex, hn, inlier_thresh, min_num, max_num, select_mode, seed, img_base, capacity):
    """(descriptor, workspace bytes) for this problem shape; only seed / img_base change between calls of a steady loop,
    so the ctypes struct and the layout query are built once per shape (the host side of a call stays ~50 us)."""
    key = (mask.dtype, mask.stride(), tuple(vertex.shape), vertex.stride(), hn, float(inlier_thresh), min_num, max_num,
           select_mode, capacity)
    hit = _desc_cache.get(key)
    if hit is None:
        d = _make_desc(mask, vertex, hn, inlier_thresh, min_num, max_num, select_mode, 0, 0, capacity)
        nbytes = lib.pvb_workspace_bytes(d)
        if nbytes == 0:
            _lib.check(lib.pvb_workspace_layout(d, _lib.PvbLayout()))
        if len(_desc_cache) > 64:
            _desc_cache.clear()
        hit = _desc_cache[key] = (d, nbytes)
    d, nbytes = hit
    d.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    d.img_base = int(img_base)
    return d, nbytes


def _make_desc(mask, vertex, hn, inlier_thresh, min_num, max_num, select_mode, seed, img_base, capacity):
    d = _lib.PvbDesc()
    d.B, d.H, d.W, d.K = vertex.size(0), vertex.size(1), vertex.size(2), vertex.size(3)
    d.hn = int(hn)
    d.inlier_thresh = float(inlier_thresh)
    d.min_num, d.max_num = int(min_num), int(min(max_num, 2 ** 31 - 1))
    d.mask_dtype = _MASK_DTYPES[mask.dtype]
    d.select_mode = select_mode
    for i in range(3):
        d.mask_stride[i] = mask.stride(i)
    for i in range(5):
        d.vertex_stride[i] = vertex.stride(i)
    d.capacity = int(capacity or 0)
    d.img_base = int(img_base)
    d.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return d


def _normal_eq(partial, tn, state, cap):
    """The refit's normal equations per (image, keypoint), float64 [B,K,5] = (a00, a01, a11, b0, b1): the first
    ceil(tn/RF_CHUNK) partials summed in split order, as the refit kernel's last CTA sums them (later splits hold data
    of earlier calls).  Skipped images give zeros."""
    nsplit = (tn.clamp(0, cap) + RF_CHUNK - 1) // RF_CHUNK
    nsplit = torch.where(state == 0, nsplit, torch.zeros_like(nsplit))
    acc = torch.zeros_like(partial[:, :, 0])
    for sp in range(int(nsplit.max())):
        use = (sp < nsplit)[:, None, None]
        acc = acc + torch.where(use, partial[:, :, sp], torch.zeros_like(acc))
    return acc


def _views(ws, d, lib, refit=False):
    """Cloned intermediates of the last call on this workspace (debug / tests); `refit`: the call ran the v3 refit."""
    L = _lib.PvbLayout()
    _lib.check(lib.pvb_workspace_layout(d, L))
    B, K, hn, cap = d.B, d.K, d.hn, L.capacity

    def view(off, count, dtype):
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return ws[off:off + nbytes].view(dtype)

    out = dict(
        tn=view(L.tn, B, torch.int32).clone(),
        state=view(L.state, B, torch.int32).clone(),
        nz=view(L.nz, B, torch.int32).clone(),
        fgsum=view(L.fgsum, B, torch.int64).clone(),
        xy=view(L.xy, B * cap * 2, torch.float32).view(B, cap, 2).clone(),
        dirs=view(L.dirs, B * K * cap * 2, torch.float32).view(B, K, cap, 2).clone(),
        hyp=view(L.hyp, B * K * hn * 2, torch.float32).view(B, K, hn, 2).clone(),
        counts=view(L.counts, B * K * hn, torch.int32).view(B, K, hn).clone(),
        win=view(L.win, B * K * 2, torch.float32).view(B, K, 2).clone(),
        capacity=cap,
    )
    if refit:
        assert L.refit_splits == (cap + RF_CHUNK - 1) // RF_CHUNK, "RF_CHUNK differs from csrc/vote.cu"
        partial = view(L.refit_partial, B * K * L.refit_splits * 5, torch.float64).view(B, K, L.refit_splits, 5)
        out["normal_eq"] = _normal_eq(partial, out["tn"], out["state"], cap)
    return out


def _torch_rng_draws(mask, hn, K, min_num, max_num, select_mode, rounds=1):
    """Consumes torch's CUDA generator exactly like the reference loop does
    (ransac_voting_gpu.py:123-145 / :205-235): per image, in order, an optional
    `uniform_` over [h,w] and then `rounds` calls of `random_(0, tn)` over [hn,K,2]."""
    B, H, W = mask.shape
    dev = mask.device
    if select_mode == _lib.PVB_SELECT_BYTE:
        cur = mask.byte() if mask.dtype != torch.bool else mask.to(torch.uint8)
        fg = cur.sum(dim=(1, 2))
    else:
        cur = (mask == 1)
        fg = cur.sum(dim=(1, 2))
    fg_host = fg.tolist()
    selection = None
    idxs = torch.zeros((B, hn * rounds, K, 2), dtype=torch.int32, device=dev)
    for bi in range(B):
        if fg_host[bi] < min_num:
            continue
        sel_mask = cur[bi] != 0
        if fg_host[bi] > max_num:
            if selection is None:
                selection = torch.ones((B, H, W), dtype=torch.float32, device=dev)
            s = torch.zeros((H, W), dtype=torch.float32, device=dev).uniform_(0, 1)
            selection[bi] = s
            sel_mask = sel_mask & (s < (max_num / fg[bi].float()))
        tn = int(sel_mask.sum().item())
        if tn == 0:
            continue
        for r in range(rounds):
            idxs[bi, r * hn:(r + 1) * hn] = torch.zeros((hn, K, 2), dtype=torch.int32, device=dev).random_(0, tn)
    return idxs, selection


def _prep_optional(t, shape, dtype, name, device):
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device:
        raise RuntimeError(f"{name} must be a CUDA tensor on the same device")
    if tuple(t.shape) != tuple(shape):
        raise RuntimeError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")
    return t.to(dtype).contiguous()


def _run(op, mask, vertex, hn, inlier_thresh, min_num, max_num, mean=None, idxs=None, selection=None,
         rng="philox", seed=None, img_base=0, capacity=None, debug=False, rounds=1, round_hn=None, exchange=None):
    mask, vertex = _check_inputs(mask, vertex)
    lib = _lib.load()
    dev = vertex.device
    B, H, W, K, _ = vertex.shape
    select_mode = _lib.PVB_SELECT_BYTE if op == "v3" else _lib.PVB_SELECT_EQ1
    if rng not in ("philox", "torch"):
        raise ValueError("rng must be 'philox' or 'torch'")
    with torch.cuda.device(dev):
        if rng == "torch" and idxs is None:
            idxs, sel = _torch_rng_draws(mask, round_hn or hn, K, min_num, max_num, select_mode, rounds)
            if selection is None:
                selection = sel
        idxs = _prep_optional(idxs, (B, hn, K, 2), torch.int32, "idxs", dev)
        selection = _prep_optional(selection, (B, H, W), torch.float32, "selection", dev)
        if seed is None:
            seed = _draw_seed() if (idxs is None or selection is None) else 0
        if capacity is None and selection is not None:
            capacity = H * W
        if capacity is not None and _VALIDATE_CAPACITY:
            # a too-small capacity would silently truncate the pixel set (the kernels clamp tn and only the sticky status
            # word, read by debug=True / pvb_read_status, says so): refuse it up front
            need = H * W if selection is not None else min(H * W, int(max_num + 8 * math.sqrt(max(max_num, 0)) + 64))
            if int(capacity) < need:
                raise RuntimeError(f"capacity={capacity} cannot hold the selection (needs >= {need}; H*W is always safe)")
        d, nbytes = _cached_desc(lib, mask, vertex, hn, inlier_thresh, min_num, max_num, select_mode, seed, img_base, capacity)
        ws = _workspace(dev, nbytes)
        stream = torch.cuda.current_stream(dev).cuda_stream
        ip = idxs.data_ptr() if idxs is not None else None
        sp = selection.data_ptr() if selection is not None else None
        if op == "v3":
            out = torch.empty((B, K, 2), dtype=torch.float32, device=dev)
            if debug and (B or exchange is not None):
                # the counts are returned: score every hypothesis (the plain entries skip those that cannot win)
                ex, seq = exchange if exchange is not None else (None, 0)
                _lib.check(lib.pvb_ransac_voting_v3_all_counts(d, mask.data_ptr(), vertex.data_ptr(), ip, sp, out.data_ptr(),
                                                               ws.data_ptr(), ws.numel(), ex, seq, stream))
            elif exchange is not None:        # (handle, seq): the refit kernel also pushes `out` to every peer
                _lib.check(lib.pvb_ransac_voting_v3_push(d, mask.data_ptr(), vertex.data_ptr(), ip, sp, out.data_ptr(),
                                                         ws.data_ptr(), ws.numel(), exchange[0], exchange[1], stream))
            elif B:
                _lib.check(lib.pvb_ransac_voting_v3(d, mask.data_ptr(), vertex.data_ptr(), ip, sp, out.data_ptr(),
                                                    ws.data_ptr(), ws.numel(), stream))
        else:
            if not isinstance(mean, torch.Tensor) or not mean.is_cuda or tuple(mean.shape) != (B, K, 2):
                raise RuntimeError("mean must be a CUDA tensor [b,vn,2]")
            mean_c = mean.float().contiguous()
            out = torch.empty((B, K, 2, 2), dtype=torch.float32, device=dev)
            if exchange is not None:
                _lib.check(lib.pvb_estimate_voting_distribution_push(d, mask.data_ptr(), vertex.data_ptr(), mean_c.data_ptr(),
                                                                     ip, sp, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                                                     exchange[0], exchange[1], stream))
            elif B:
                _lib.check(lib.pvb_estimate_voting_distribution(d, mask.data_ptr(), vertex.data_ptr(),
                                                                mean_c.data_ptr(), ip, sp, out.data_ptr(),
                                                                ws.data_ptr(), ws.numel(), stream))
        if debug:
            if B:
                _lib.check(lib.pvb_read_status(d, ws.data_ptr(), stream))
            info = _views(ws, d, lib, refit=(op == "v3")) if B else {}
            info["seed"] = seed
            return out, info
    return out


def ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                           min_num=5, max_num=30000, *, idxs=None, selection=None, rng="philox", seed=None,
                           img_base=0, capacity=None, debug=False, _exchange=None):
    """Drop-in for ransac_voting_gpu.py:112-199.

    :param mask:      [b,h,w]   any integer / bool / float dtype, any strides
    :param vertex:    [b,h,w,vn,2] float32, any strides (e.g. the permuted NCHW view of resnet18.py:66-68)
    :param round_hyp_num: hypotheses per (image, keypoint)
    :param inlier_thresh: cosine threshold
    :return: [b,vn,2] float32 on mask.device

    `confidence` and `max_iter` are accepted for signature compatibility.  In the reference the
    sample pairs are drawn once, before the `while True` loop (:145 vs :150), so every extra round
    re-scores identical hypotheses and the result equals that of round one; one round is run here.
    """
    del confidence, max_iter
    return _run("v3", mask, vertex, int(round_hyp_num), inlier_thresh, min_num, max_num, idxs=idxs,
                selection=selection, rng=rng, seed=seed, img_base=img_base, capacity=capacity, debug=debug,
                exchange=_exchange)


def ransac_voting_layer(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                        min_num=5, max_num=30000, **kw):
    """Drop-in for ransac_voting_gpu.py:6-95 (imported by resnet18.py:5, never called there).
    v1 differs from v3 only in how a singular 2x2 normal matrix is handled (torch.inverse in a
    try/except -> zeros for the whole image, :86-91, vs b_inv's identity, :105-108); both code
    paths are degenerate (no inliers) and this implementation returns ATb (= 0) for that keypoint."""
    return ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh, confidence, max_iter,
                                  min_num, max_num, **kw)


def estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=256, min_hyp_num=4096, topk=128,
                                           inlier_thresh=0.99, min_num=5, max_num=30000, output_hyp=False, *,
                                           idxs=None, selection=None, rng="philox", seed=None, img_base=0,
                                           capacity=None, debug=False, _exchange=None):
    """Drop-in for ransac_voting_gpu.py:202-274: returns (mean, cov[b,vn,2,2]).
    `topk` and `output_hyp` are unused by the reference as well."""
    del topk, output_hyp
    rounds = int(math.ceil(min_hyp_num / round_hyp_num))
    hn = int(round_hyp_num) * rounds
    res = _run("dist", mask, vertex, hn, inlier_thresh, min_num, max_num, mean=mean, idxs=idxs,
               selection=selection, rng=rng, seed=seed, img_base=img_base, capacity=capacity, debug=debug,
               rounds=rounds, round_hn=int(round_hyp_num), exchange=_exchange)
    if debug:
        return mean, res[0], res[1]
    return mean, res


# ---------------------------------------------------------------------------------------------
# host-buffer entry (end-to-end path: pinned host tensors in, host tensor out)
# ---------------------------------------------------------------------------------------------
_host_scratch = {}


def ransac_voting_layer_v3_host(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                                min_num=5, max_num=30000, *, device=None, chunk_images=4, seed=None, img_base=0,
                                out=None, mode="auto"):
    """ransac_voting_layer_v3 for HOST tensors: the C ABI's host-buffer entry (pvb_ransac_voting_v3_host)
    processes the batch in `chunk_images`-sized pieces on three streams and writes keypoints to a host tensor.
    mode (what crosses PCIe, see include/pvnet_vote_b200.h):
        "auto"     pinned inputs: the mask goes by DMA (one cudaMemcpyAsync per piece), the vertex field is read in place and
                   only the selected pixels' rows cross the bus (tn*K*8 bytes per image instead of the dense H*W*K*8);
                   pageable inputs are staged
        "inplace"  both tensors read in place by the kernels (no DMA)
        "staged"   both tensors copied with cudaMemcpyAsync"""
    del confidence, max_iter
    if mask.is_cuda or vertex.is_cuda:
        raise RuntimeError("ransac_voting_layer_v3_host takes host tensors")
    if vertex.dtype != torch.float32 or not vertex.is_contiguous() or not mask.is_contiguous():
        raise RuntimeError("host path needs contiguous float32 vertex and contiguous mask")
    if mask.dtype not in _MASK_DTYPES:
        raise RuntimeError(f"unsupported mask dtype {mask.dtype}")
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    B, H, W, K, _ = vertex.shape
    if seed is None:
        seed = _draw_seed()
    d = _make_desc(mask, vertex, int(round_hyp_num), inlier_thresh, min_num, max_num, _lib.PVB_SELECT_BYTE, seed,
                   img_base, None)
    chunk = max(1, min(int(chunk_images), B)) if B else 1
    if out is None:
        out = torch.empty((B, K, 2), dtype=torch.float32).pin_memory()
    if B == 0:
        return out
    with torch.cuda.device(dev):
        nbytes = lib.pvb_host_scratch_bytes(d, chunk)
        key = dev.index
        sc = _host_scratch.get(key)
        if sc is None or sc.numel() < nbytes:
            sc = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
            _host_scratch[key] = sc
        flags = {"auto": 0, "inplace": _lib.PVB_HOST_INPLACE_MASK, "staged": _lib.PVB_HOST_STAGE_VERTEX}[mode]
        _lib.check(lib.pvb_ransac_voting_v3_host(d, mask.data_ptr(), vertex.data_ptr(), out.data_ptr(), chunk, flags,
                                                 sc.data_ptr(), sc.numel(),
                                                 torch.cuda.current_stream(dev).cuda_stream))
    return out


def install_as_reference_module():
    """Makes `from lib.csrc.ransac_voting.ransac_voting_gpu import ...` (lib/networks/pvnet/resnet18.py:5) resolve to
    this module, and `import lib.csrc.ransac_voting.ransac_voting` (ransac_voting_gpu.py:2) to the twins of the pybind
    extension -- WITHOUT shadowing anything else of the reference tree.

    Only the two leaf modules are replaced.  The parents `lib`, `lib.csrc`, `lib.csrc.ransac_voting` are the REAL
    packages whenever they can be imported (the normal case: the call sits at the top of run.py / train_net.py with
    the clean-pvnet checkout on sys.path), so `lib.config`, `lib.networks`, `lib.csrc.nn`, `lib.csrc.uncertainty_pnp`
    keep importing.  A stand-in package is created only for a parent that does not exist anywhere on sys.path
    (using this module outside a clean-pvnet checkout).  Idempotent."""
    from ._dropin import reference_package
    this = sys.modules[__name__]
    parent = reference_package("lib.csrc.ransac_voting")
    sys.modules["lib.csrc.ransac_voting.ransac_voting_gpu"] = this
    sys.modules["lib.csrc.ransac_voting.ransac_voting"] = _ext
    parent.ransac_voting_gpu = this
    parent.ransac_voting = _ext
    return this
