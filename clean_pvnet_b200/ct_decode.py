"""The CenterNet detector's decode on the device, from its output maps to image-frame boxes (DESIGN.md section 8j; the
kernels are csrc/ct_decode.cu):

    decode_detections(ct_hm, wh, K, clip)      Network.decode_detection (lib/networks/ct/dla.py:20-26) for B images:
                                               sigmoid, decode_ct_hm and clip_to_image -> (ct [B,K,2], detection [B,K,6])
    detection_boxes(detection, center, scale, input_size, down_ratio)
                                               every consumer's affine_transform(box * down_ratio,
                                               get_affine_transform(center, scale, 0, [w, h], inv=1)) -> [B,K,4] f64
    install_ct_decode_as_reference()           `lib.networks.ct.dla.Network.decode_detection` runs on the device

With crop.crop_inputs and crop.uncrop_keypoints this takes T-LESS inference from the detector's raw maps to PVNet's
inputs and back for a whole batch, with no host step.
"""
import ctypes
import importlib

import torch

from . import _lib
from .nn import _call, _workspace


def _strides(t):
    return (ctypes.c_int64 * 4)(*[int(s) for s in t.stride()])


def decode_detections(ct_hm, wh, K=100, clip=True):
    """Network.decode_detection's two tensors for all B images (lib/networks/ct/dla.py:20-26): ct_decode.decode_ct_hm
    (lib/utils/ct/ct_decode.py:6-75) of torch.sigmoid(ct_hm), then, with clip, data_utils.clip_to_image to the map's
    H x W.  ct_hm: float32 [B,C,H,W] CUDA logits, wh: float32 [B,2,H,W] on the same device, any strides (channels-last
    included).  Returns (ct float32 [B,K,2] (xs, ys), detection float32 [B,K,6] (x0, y0, x1, y1, score, class)), equal
    to CUDA torch's bit for bit, with equal scores ordered by class and then by pixel index.  Runs on the current stream,
    never waits for the device and can be captured in a CUDA graph.  Bad input raises RuntimeError before any launch."""
    for name, t in (("ct_hm", ct_hm), ("wh", wh)):
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise RuntimeError(f"{name} must be a CUDA tensor")
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32 (the detector's output), got {t.dtype}")
    if ct_hm.dim() != 4:
        raise RuntimeError(f"ct_hm must be [B,C,H,W], got {list(ct_hm.shape)}")
    B, C, H, W = (int(s) for s in ct_hm.shape)
    if tuple(wh.shape) != (B, 2, H, W):
        raise RuntimeError(f"wh must be [{B},2,{H},{W}], got {list(wh.shape)}")
    if wh.device != ct_hm.device:
        raise RuntimeError(f"ct_hm and wh must be on one device, got {ct_hm.device} and {wh.device}")
    if isinstance(K, bool) or not isinstance(K, int):
        raise RuntimeError(f"K must be an int, got {K!r}")
    if C < 1 or H < 1 or W < 1:
        raise RuntimeError(f"ct_hm must have C, H, W >= 1, got {list(ct_hm.shape)}")
    if H * W >= 1 << 24:
        raise RuntimeError(f"H*W must be < 2^24 (the reference's fp32 row index is exact below it), got {H * W}")
    if not 1 <= K <= H * W:
        raise RuntimeError(f"K must be in [1, H*W = {H * W}] (torch.topk raises above it), got {K}")
    if C * K >= 1 << 24:
        raise RuntimeError(f"C*K must be < 2^24 (the reference's fp32 class index is exact below it), got {C * K}")
    dev = ct_hm.device
    ct = torch.empty((B, K, 2), dtype=torch.float32, device=dev)
    det = torch.empty((B, K, 6), dtype=torch.float32, device=dev)
    if B == 0:
        return ct, det
    nbytes = _lib.load().pvb_ct_decode_workspace_bytes(B, C, H, W, K)
    ws = _workspace(nbytes, dev)
    _call("pvb_ct_decode", dev, ct_hm, _strides(ct_hm), wh, _strides(wh), B, C, H, W, K, int(bool(clip)), ct, det,
          ws, nbytes)
    return ct, det


def detection_boxes(detection, center, scale, input_size, down_ratio=4):
    """The image-frame boxes every consumer of the decode computes on the host, one image at a time (the cascade's
    res.crop, lib/networks/ct_pvnet/res.py:35-57, and the evaluator, lib/evaluators/tless_test/ct.py:33-60):
        affine_transform((box * down_ratio).reshape(-1, 2), get_affine_transform(center, scale, 0, [w, h], inv=1))
    for every row of every image.  detection [B,K,>=4] float32 (decode_detections' output), center [B,2] and scale [B]
    or [B,2] (batch['meta']'s; like get_affine_transform, only scale[:, 0] is used), input_size (w, h) of the detector's
    input.  Returns float64 [B,K,4] (x0, y0, x1, y1) on the device of detection, within 1e-12 px of the reference.  The
    un-crop kernel builds the matrix from scale rounded to float32, so a scale that float32 cannot represent exactly is
    refused (the datasets' max(H, W) always can); checking a float64 CUDA scale waits for the device."""
    d = torch.as_tensor(detection)
    if d.dim() != 3 or d.shape[2] < 4:
        raise RuntimeError(f"detection must be [B,K,>=4], got {list(d.shape)}")
    B, K = int(d.shape[0]), int(d.shape[1])
    c, s = torch.as_tensor(center), torch.as_tensor(scale)
    if tuple(c.shape) != (B, 2):
        raise RuntimeError(f"center must be [{B},2], got {list(c.shape)}")
    if s.dim() == 2 and s.shape[1] == 2:
        s = s[:, 0]
    if tuple(s.shape) != (B,):
        raise RuntimeError(f"scale must be [{B}] or [{B},2], got {list(torch.as_tensor(scale).shape)}")
    s64 = s.to(torch.float64)
    if not bool((s64.to(torch.float32).to(torch.float64) == s64).all()):
        raise RuntimeError("scale must be exactly representable in float32 (the un-crop builds its matrix from float32 "
                           "scale); the datasets' max(H, W) always is")
    w, h = (int(v) for v in input_size)
    if w < 1 or h < 1:
        raise RuntimeError(f"input_size must be (width, height) >= 1, got {input_size}")
    dev = d.device if d.is_cuda else torch.device("cuda", torch.cuda.current_device())
    kpt = (d[..., :4].to(device=dev, dtype=torch.float32) * down_ratio).reshape(B, 2 * K, 2).contiguous()
    c = c.to(device=dev, dtype=torch.float64).contiguous()
    s64 = s64.to(dev).contiguous()
    out = torch.empty((B, 2 * K, 2), dtype=torch.float64, device=dev)
    if B and K:
        _call("pvb_uncrop_keypoints", dev, kpt, c, s64, B, 2 * K, w, h, out)
    return out.reshape(B, K, 4)


def _decode_detection(self, output, h, w):
    """Network.decode_detection on the device: the same output['ct'] / output['detection'] and return value."""
    ct_hm, wh = output['ct_hm'], output['wh']
    if (int(h), int(w)) != tuple(int(v) for v in ct_hm.shape[2:]):
        raise RuntimeError(f"decode_detection clips to the heatmap's own size; got h, w = {h}, {w} for a "
                           f"{list(ct_hm.shape)} heatmap")
    ct, detection = decode_detections(ct_hm.detach(), wh.detach())
    output.update({'ct': ct, 'detection': detection})
    return ct, detection


def install_ct_decode_as_reference():
    """Makes the detector (lib/networks/ct/dla.py Network) decode its output on the device: only
    Network.decode_detection is replaced, so the detector, the detector -> PVNet cascade (lib/networks/ct_pvnet/res.py
    builds its detector from ct.dla) and the detection evaluator run unchanged on the fused decode.  Importing ct.dla
    imports the DCN layers, so call install_dcn_as_reference_module() first.  Idempotent; coexists with
    install_crop_as_reference() in either order.  Returns the patched module."""
    from ._dropin import reference_package
    reference_package("lib.networks.ct")
    dla = importlib.import_module("lib.networks.ct.dla")
    dla.Network.decode_detection = _decode_detection
    return dla
