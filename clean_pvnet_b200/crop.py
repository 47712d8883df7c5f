"""T-LESS's PVNet crop on the device (DESIGN.md section 8g; the kernels are csrc/crop.cu):

    crop_inputs(img, boxes, ...)                 tless_test_utils.pvnet_transform (lib/utils/tless/tless_test_utils.py:
                                                 57-77) for n boxes -> (inp [n,3,h,w] f32, center [n,2] f32, scale [n] f32)
    uncrop_keypoints(kpt_2d, center, scale, input_size)
                                                 the evaluator's affine_transform(kpt, get_affine_transform(..., inv=1))
                                                 (lib/evaluators/tless_test/pvnet.py:229-239) -> [n,K,2] f64
    warp_affine_batch(img, M, dsize)             cv2.warpAffine(img, M, dsize, flags=INTER_LINEAR) for n rows
    install_crop_as_reference()                  `lib.networks.ct_pvnet.res.crop` (the cascade's crop) runs on the device

Pixels are cv2.warpAffine's byte for byte and the crop matrices cv2.getAffineTransform's bit for bit; nothing waits for
the device and the image never leaves it.
"""
import ctypes
import importlib
import sys

import numpy as np
import torch

from . import _lib
from .nn import _call

# lib/utils/tless/tless_config.py
MEAN = (0.40789654, 0.44719302, 0.47026115)
STD = (0.28863828, 0.27408164, 0.27809835)


def _device(*ts):
    for t in ts:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            return t.device
    return torch.device("cuda", torch.cuda.current_device())


def _images(img, channels=None):
    """img [H,W,C] or [B,H,W,C] uint8, any strides -> ([B,H,W,C] tensor, B, H, W, C), checked before anything moves."""
    t = torch.as_tensor(img)
    if t.dtype != torch.uint8 or t.dim() not in (3, 4) or (channels is not None and t.shape[-1] != channels):
        want = f"[H,W,{channels}] or [B,H,W,{channels}]" if channels else "[H,W,C] or [B,H,W,C]"
        raise RuntimeError(f"img must be a uint8 {want} tensor, got {t.dtype} {list(t.shape)}")
    if t.dim() == 3:
        t = t.unsqueeze(0)
    B, H, W, C = (int(s) for s in t.shape)
    return t, B, H, W, C


def _strides(t):
    return (ctypes.c_int64 * 4)(*[int(s) for s in t.stride()])


def _index(image_index, n, B):
    if image_index is None:
        if B != 1:
            raise RuntimeError(f"image_index is required when img holds {B} images")
        return None
    ix = torch.as_tensor(image_index)
    if ix.dim() != 1 or int(ix.shape[0]) != n or ix.dtype.is_floating_point or ix.dtype == torch.bool:
        raise RuntimeError(f"image_index must be an integer [{n}] tensor, got {ix.dtype} {list(ix.shape)}")
    return ix


def _size(size, name):
    w, h = (int(s) for s in size)
    if w < 1 or h < 1:
        raise RuntimeError(f"{name} must be (width, height) >= 1, got {size}")
    return w, h


def _floats3(v):
    return (ctypes.c_float * 3)(*[float(x) for x in np.asarray(v, np.float32).reshape(3)])


def crop_device(img, boxes, image_index=None, input_size=(256, 256), scale_ratio=2.4, box_ratio=1.2, mask_to_box=True,
                center_f64=False, return_uint8=False, mean=MEAN, std=STD):
    """pvb_crop_inputs: (inp, crop_u8 or None, center f64 [n,2], scale f64 [n], matrix [n,2,3], matrix_inv [n,2,3])."""
    b = torch.as_tensor(boxes)
    if b.dim() != 2 or b.shape[1] != 4:
        raise RuntimeError(f"boxes must be [n,4] (x0, y0, x2, y2), got {list(b.shape)}")
    w, h = _size(input_size, "input_size")
    im, B, H, W, _ = _images(img, 3)
    n = int(b.shape[0])
    ix = _index(image_index, n, B)
    dev = _device(im, b)
    im = im.to(dev)
    ix = None if ix is None else ix.to(device=dev, dtype=torch.int32).contiguous()
    b = b.to(device=dev, dtype=torch.float64).contiguous()
    f64 = dict(dtype=torch.float64, device=dev)
    inp = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
    u8 = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev) if return_uint8 else None
    center, scale = torch.empty((n, 2), **f64), torch.empty((n,), **f64)
    M, Minv = torch.empty((n, 2, 3), **f64), torch.empty((n, 2, 3), **f64)
    flags = (_lib.PVB_CROP_MASK_TO_BOX if mask_to_box else 0) | (_lib.PVB_CROP_CENTER_F64 if center_f64 else 0)
    _call("pvb_crop_inputs", dev, im, B, H, W, _strides(im), b, ix, n, w, h, float(scale_ratio), float(box_ratio), flags,
          _floats3(mean), _floats3(std), inp, u8, center, scale, M, Minv)
    return inp, u8, center, scale, M, Minv


def crop_inputs(img, boxes, image_index=None, input_size=(256, 256), scale_ratio=2.4, box_ratio=1.2, mask_to_box=True,
                return_uint8=False, mean=MEAN, std=STD):
    """tless_test_utils.pvnet_transform(img, box) (lib/utils/tless/tless_test_utils.py:57-77) for n boxes at once.
        img          uint8 [H,W,3] or [B,H,W,3] BGR, any strides (a CUDA tensor stays where it is; anything else is copied
                     to the current CUDA device once)
        boxes        [n,4] xyxy in image coordinates, used in float64
        image_index  integer [n]: the image of each box (required when img holds more than one image)
        input_size   (width, height) of the crop, as cv2's dsize and as pvnet_transform unpacks input_scale (the cascade's
                     res.py unpacks it as (height, width); T-LESS's (256, 256) is square)
        scale_ratio, box_ratio, mean, std    cfg.tless's scale_ratio / box_ratio and T-LESS's normalisation
        mask_to_box  zero what lies outside magnify_box(box, box_ratio) (pvnet_transform does; the cascade's _crop not)
    Returns (inp float32 [n,3,h,w], center float32 [n,2], scale float32 [n][, crop uint8 [n,h,w,3]]) on the device:
    inp and crop (the dataset's orig_img) equal pvnet_transform's bit for bit; center is its float32 centre and scale its
    max(w, h) * scale_ratio rounded to float32, which is what get_affine_transform builds the matrix from.  Nothing
    waits for the device."""
    inp, u8, center, scale, _, _ = crop_device(img, boxes, image_index, input_size, scale_ratio, box_ratio, mask_to_box,
                                               False, return_uint8, mean, std)
    out = (inp, center.float(), scale.float())
    return out + (u8,) if return_uint8 else out


def uncrop_keypoints(kpt_2d, center, scale, input_size=(256, 256)):
    """The evaluator's un-crop (lib/evaluators/tless_test/pvnet.py:229-239), affine_transform(kpt_2d[i],
    get_affine_transform(center[i], scale[i], 0, input_size, inv=1)), for n boxes: kpt_2d [n,K,2] in the crop frame
    (rounded to float32, as the network emits it), center [n,2] and scale [n] as crop_inputs returns them (or the
    reference's float64 values), input_size (width, height).  Returns float64 [n,K,2] image coordinates on the device of
    kpt_2d, ready for pnp_batch / uncertainty_pnp_from_votes; within 1e-12 px of the reference."""
    k, c, s = torch.as_tensor(kpt_2d), torch.as_tensor(center), torch.as_tensor(scale)
    if k.dim() != 3 or k.shape[2] != 2:
        raise RuntimeError(f"kpt_2d must be [n,K,2], got {list(k.shape)}")
    n, K = int(k.shape[0]), int(k.shape[1])
    if tuple(c.shape) != (n, 2) or tuple(s.shape) != (n,):
        raise RuntimeError(f"center must be [{n},2] and scale [{n}], got {list(c.shape)} and {list(s.shape)}")
    w, h = _size(input_size, "input_size")
    dev = _device(k, c, s)
    k = k.to(device=dev, dtype=torch.float32).contiguous()
    c, s = (t.to(device=dev, dtype=torch.float64).contiguous() for t in (c, s))
    out = torch.empty((n, K, 2), dtype=torch.float64, device=dev)
    _call("pvb_uncrop_keypoints", dev, k, c, s, n, K, w, h, out)
    return out


def warp_affine_batch(img, M, dsize, image_index=None):
    """cv2.warpAffine(img[image_index[i]], M[i], dsize, flags=cv2.INTER_LINEAR) (zero border) for n rows, byte for byte:
    img uint8 [H,W], [H,W,C] or [B,H,W,C] with C <= 4, any strides; M [n,2,3] or [2,3] forward matrices (float64);
    dsize (width, height).  Returns uint8 [n,h,w,C] ([n,h,w] for a [H,W] image) on the device.  Covers the detector's
    full-image resize of tless_test_utils.augment as well as crops."""
    t = torch.as_tensor(img)
    gray = t.dim() == 2
    if gray:
        t = t.unsqueeze(-1)
    m = torch.as_tensor(M)
    if m.dim() == 2:
        m = m.unsqueeze(0)
    if m.dim() != 3 or tuple(m.shape[1:]) != (2, 3):
        raise RuntimeError(f"M must be [n,2,3] or [2,3], got {list(torch.as_tensor(M).shape)}")
    w, h = _size(dsize, "dsize")
    im, B, H, W, C = _images(t)
    n = int(m.shape[0])
    ix = _index(image_index, n, B)
    dev = _device(im, m)
    im = im.to(dev)
    ix = None if ix is None else ix.to(device=dev, dtype=torch.int32).contiguous()
    m = m.to(device=dev, dtype=torch.float64).contiguous()
    out = torch.empty((n, h, w, C), dtype=torch.uint8, device=dev)
    _call("pvb_warp_affine_linear", dev, im, B, H, W, C, _strides(im), m, ix, n, w, h, out)
    return out[..., 0] if gray else out


# ---- the detector -> PVNet cascade's crop (lib/networks/ct_pvnet/res.py:14-57) ---------------------------------------

def cascade_crop(img, detection, batch, output):
    """Twin of res.crop: the same boxes, centres, scales and inputs, but the image is warped on the device it is on and
    the inputs never leave it.  The only copy to the host is the one the reference makes of the detection box (after the
    score cut); the box goes through trans_output_inv there exactly as res._crop does, and back as 32 bytes."""
    res = sys.modules["lib.networks.ct_pvnet.res"]
    du, tc, tp = res.data_utils, res.tless_config, res.tless_pvnet_utils
    img = img[0].detach()
    if img.dtype != torch.uint8:
        img = img.to(torch.uint8)                    # img.astype(np.uint8), for in-range values
    max_det, ct_score, down_ratio = 1, 0, 4          # res.crop's fx_config
    box = output['detection'][0, :max_det, :4]
    score = output['detection'][0, :max_det, 4]
    box = box[score > ct_score]
    box = box.detach().cpu().numpy() * down_ratio

    center = batch['meta']['center'][0].detach().cpu().numpy()
    scale = batch['meta']['scale'][0].detach().cpu().numpy()
    h, w = batch['inp'].size(2), batch['inp'].size(3)
    trans_output_inv = du.get_affine_transform(center, scale, 0, [w, h], inv=1)
    if len(box) == 0:
        output.update({'inp': [], 'center': [], 'scale': []})
        return []
    boxes = np.stack([du.affine_transform(b.reshape(-1, 2), trans_output_inv).ravel() for b in box])
    centers = tuple(np.array([(b[0] + b[2]) / 2, (b[1] + b[3]) / 2]) for b in boxes)
    scales = tuple(max(b[2] - b[0], b[3] - b[1]) * tc.scale_ratio for b in boxes)
    input_h, input_w = tp.input_scale
    dev = img.device if img.is_cuda else torch.device("cuda", torch.cuda.current_device())
    inp = crop_device(img, torch.from_numpy(boxes).to(dev), None, (int(input_w), int(input_h)), float(tc.scale_ratio),
                      0.0, False, True, False, np.asarray(tc.mean).reshape(3), np.asarray(tc.std).reshape(3))[0]
    output.update({'inp': inp, 'center': centers, 'scale': scales})
    return inp


def install_crop_as_reference():
    """Makes the detector -> PVNet cascade (lib/networks/ct_pvnet/res.py, Network.forward) crop on the device: only
    `lib.networks.ct_pvnet.res.crop` is replaced (by cascade_crop); the module itself, `_crop`, `Network` and every other
    `lib.*` module stay the real ones.  Idempotent.  Returns the patched module."""
    from ._dropin import reference_package
    reference_package("lib.networks.ct_pvnet")
    res = importlib.import_module("lib.networks.ct_pvnet.res")
    res.crop = cascade_crop
    return res
