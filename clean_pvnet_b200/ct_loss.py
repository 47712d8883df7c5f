"""The CenterNet detector's heatmap target and focal loss computed from its boxes on the device, so detector training
never ships the dense [30,H,W] heatmap per sample (DESIGN.md section 8i; the kernels are csrc/ct_loss.cu):

    ct_radius(wh)                          the datasets' radius rule, max(0, int(gaussian_radius((ceil(h), ceil(w))))),
                                           on the sample's float64 box sizes
    ct_target_batch(...)                   the datasets' ct_hm (data_utils.draw_umich_gaussian per object) for B images,
                                           float32 [B,C,H,W], bit for bit
    ct_focal_loss(logits, ...)             the trainer's FocalLoss(net_utils.sigmoid(logits), ct_hm) with that target, an
                                           autograd Function; its gradient for the logits is autograd's bit for bit
    CtNetworkWrapper(net)                  twin of lib/train/trainers/ct.py's NetworkWrapper on ct_focal_loss
    install_ct_loss_as_reference()         the zero-edit drop-in for clean-pvnet's collator and trainer

An image's objects are four [B,M] arrays, as the collator pads them: ct_ind (cy * W + cx), ct_radius, ct_cls and ct_01
(1 for an object, 0 for padding).
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib
from .nn import _call, _workspace

MAX_OBJECTS = 1024        # objects per image the kernels stage in shared memory (pvb_ct_* reject more)


def _gaussian_radius(height, width, min_overlap=0.7):
    """data_utils.gaussian_radius (lib/utils/data_utils.py:10-33) of integer height and width: the smallest of the three
    quadratic roots, each term in the reference's operation order (Python floats, so every rounding is the same)."""
    s = height + width
    hw = width * height
    r1 = (s + np.sqrt(s ** 2 - 4 * 1 * (hw * (1 - min_overlap) / (1 + min_overlap)))) / 2
    r2 = (2 * s + np.sqrt((2 * s) ** 2 - 4 * 4 * ((1 - min_overlap) * width * height))) / 2
    a3, b3, c3 = 4 * min_overlap, -2 * min_overlap * s, (min_overlap - 1) * width * height
    disc = b3 ** 2 - 4 * a3 * c3
    r3 = min(r1, r2) if disc < 0 else (b3 + np.sqrt(disc)) / 2
    return min(r1, r2, r3)


def ct_radius(wh):
    """The radius every CenterNet dataset draws an object with (lib/datasets/tless*/ct.py prepare_detection):
    max(0, int(gaussian_radius((ceil(h), ceil(w))))).  wh: [..., 2] of (w, h), the sample's own float64 sizes (the
    batch's float32 wh can round a size just above an integer down onto it).  Returns int32 [...]."""
    wh = np.asarray(wh, np.float64)
    if wh.shape[-1:] != (2,):
        raise ValueError(f"wh must be [..., 2] (w, h), got {wh.shape}")
    flat = wh.reshape(-1, 2)
    out = [max(0, int(_gaussian_radius(math.ceil(h), math.ceil(w)))) for w, h in flat.tolist()]
    return np.asarray(out, np.int32).reshape(wh.shape[:-1])


def _objects(ct_ind, ct_radius, ct_cls, ct_01, dev):
    """The four [B,M] object arrays as contiguous device tensors of the kernels' dtypes (int64, int32, int64, float32)."""
    arrays = []
    for name, a, dt in (("ct_ind", ct_ind, torch.int64), ("ct_radius", ct_radius, torch.int32),
                        ("ct_cls", ct_cls, torch.int64), ("ct_01", ct_01, torch.float32)):
        t = torch.as_tensor(a)
        if t.dim() != 2:
            raise RuntimeError(f"{name} must be [B,M], got {list(t.shape)}")
        if t.is_floating_point() and dt != torch.float32:
            raise RuntimeError(f"{name} must be an integer tensor, got {t.dtype}")
        arrays.append(t.to(device=dev, dtype=dt).contiguous())
    shape = arrays[0].shape
    if any(a.shape != shape for a in arrays):
        raise RuntimeError(f"ct_ind, ct_radius, ct_cls and ct_01 must share one [B,M] shape, got "
                           f"{[list(a.shape) for a in arrays]}")
    if shape[1] > MAX_OBJECTS:
        raise RuntimeError(f"at most {MAX_OBJECTS} objects per image, got M = {shape[1]}")
    return arrays


def ct_target_batch(ct_ind, ct_radius, ct_cls, ct_01, num_classes, height, width, device=None):
    """The ct_hm the CenterNet datasets draw (data_utils.draw_umich_gaussian per object, lib/utils/data_utils.py:36-64),
    for B images at once, bit for bit: float32 [B,num_classes,height,width] on `device` (default: ct_ind's device, which
    must be a CUDA device).  The objects are [B,M] arrays (tensors or numpy) as the collator pads them."""
    dev = torch.device(device) if device is not None else torch.as_tensor(ct_ind).device
    if dev.type != "cuda":
        raise RuntimeError("ct_target_batch runs on a CUDA device: pass CUDA tensors or device='cuda'")
    ind, rad, cls, c01 = _objects(ct_ind, ct_radius, ct_cls, ct_01, dev)
    B, M = (int(s) for s in ind.shape)
    out = torch.empty((B, int(num_classes), int(height), int(width)), dtype=torch.float32, device=dev)
    _call("pvb_ct_target", dev, ind, rad, cls, c01, out, B, M, int(num_classes), int(height), int(width))
    return out


class _CtFocalLoss(torch.autograd.Function):
    """FocalLoss(clamp(sigmoid(logits), 1e-4, 1 - 1e-4), ct_hm) with ct_hm computed per pixel from the objects."""

    @staticmethod
    def forward(ctx, logits, ind, rad, cls, c01):
        dev = logits.device
        B, C, H, W = (int(s) for s in logits.shape)
        M = int(ind.shape[1])
        ls = (ctypes.c_int64 * 4)(*logits.stride())
        loss = torch.empty((), dtype=torch.float32, device=dev)
        nbytes = _lib.load().pvb_ct_loss_workspace_bytes(B, C, H, W)
        ws = _workspace(nbytes, dev)                       # keeps num_pos for backward
        _call("pvb_ct_loss_forward", dev, ctypes.c_void_p(logits.data_ptr() or None), ls, ind, rad, cls, c01, loss,
              B, M, C, H, W, ws, nbytes)
        ctx.save_for_backward(logits, ind, rad, cls, c01)
        ctx.ws, ctx.nbytes = ws, nbytes
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        logits, ind, rad, cls, c01 = ctx.saved_tensors
        dev = logits.device
        B, C, H, W = (int(s) for s in logits.shape)
        M = int(ind.shape[1])
        ls = (ctypes.c_int64 * 4)(*logits.stride())
        g = grad_loss.to(device=dev, dtype=torch.float32).contiguous()
        grad = torch.empty((B, C, H, W), dtype=torch.float32, device=dev)
        _call("pvb_ct_loss_backward", dev, ctypes.c_void_p(logits.data_ptr() or None), ls, ind, rad, cls, c01, g, grad,
              B, M, C, H, W, ctx.ws, ctx.nbytes)
        return grad, None, None, None, None


def ct_focal_loss(logits, ct_ind, ct_radius, ct_cls, ct_01):
    """The detector's heatmap loss of clean-pvnet's trainer (lib/train/trainers/ct.py:20-21),
        net_utils.FocalLoss()(net_utils.sigmoid(logits), ct_hm)
    with ct_hm computed per pixel on the device from the objects and never stored.  logits: float32 [B,C,H,W] CUDA
    tensor, any strides (channels-last included; other dtypes are refused); the objects: [B,M] (ct_ind int64, ct_radius
    int32, ct_cls int64, ct_01 float; CUDA tensors avoid a host copy).  Returns a 0-dim float32 tensor with a gradient for
    the logits only.  Neither pass synchronises with the host (num_pos stays on the device), and both run on the current
    stream of the logits' device, so the function works in DataParallel replicas.  The loss is reproducible bit for bit
    and within one fp32 ulp of the same chain on float64 sums of the terms; the gradient equals autograd's of the
    reference expression bit for bit."""
    if not (isinstance(logits, torch.Tensor) and logits.is_cuda):
        raise RuntimeError("logits must be a CUDA tensor")
    if logits.dtype != torch.float32:
        raise RuntimeError(f"logits must be float32 (the reference trains in fp32), got {logits.dtype}")
    if logits.dim() != 4:
        raise RuntimeError(f"logits must be [B,C,H,W], got {list(logits.shape)}")
    ind, rad, cls, c01 = _objects(ct_ind, ct_radius, ct_cls, ct_01, logits.device)
    if ind.shape[0] != logits.shape[0]:
        raise RuntimeError(f"the objects must be [B,M] with B = {logits.shape[0]}, got {list(ind.shape)}")
    return _CtFocalLoss.apply(logits, ind, rad, cls, c01)


def _ind_smooth_l1(output, target, ind, weight):
    """net_utils.IndL1Loss1d('smooth_l1') (lib/utils/net_utils.py:232-246): smooth_l1 between output's [B,D] vector at
    each object's centre and its target [B,M,D], both times the object weight, summed over the batch and divided by
    weight.sum() * D + 1e-4.  Gathers the 2*M values straight from the [B,D,H,W] map."""
    B, D = output.shape[:2]
    idx = ind[:, None, :].expand(B, D, ind.shape[1])
    feat = output.reshape(B, D, -1).gather(2, idx).transpose(1, 2)           # [B,M,D]
    w = weight.unsqueeze(2)
    loss = torch.nn.functional.smooth_l1_loss(feat * w, target * w, reduction='sum')
    return loss / (w.sum() * feat.size(2) + 1e-4)


class CtNetworkWrapper(torch.nn.Module):
    """Twin of clean-pvnet's lib/train/trainers/ct.py NetworkWrapper: the same scalar_stats keys (ct_loss, wh_loss,
    loss) and the same 0.1 weight of the size loss, with the heatmap loss computed by ct_focal_loss from the batch's
    objects (ct_ind, ct_radius, ct_cls, ct_01) instead of a dense batch['ct_hm']."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, batch):
        if 'ct_radius' not in batch:
            raise RuntimeError(
                "the batch has no 'ct_radius': call clean_pvnet_b200.install_ct_loss_as_reference() before the data "
                "loaders are built, so that the 'ct' collator passes each object's radius instead of the dense ct_hm")
        output = self.net(batch['inp'])

        scalar_stats = {}
        loss = 0

        ct_loss = ct_focal_loss(output['ct_hm'], batch['ct_ind'], batch['ct_radius'], batch['ct_cls'], batch['ct_01'])
        scalar_stats.update({'ct_loss': ct_loss})
        loss += ct_loss

        wh_loss = _ind_smooth_l1(output['wh'], batch['wh'], batch['ct_ind'], batch['ct_01'])
        scalar_stats.update({'wh_loss': wh_loss})
        loss += 0.1 * wh_loss

        scalar_stats.update({'loss': loss})
        image_stats = {}

        return output, loss, scalar_stats, image_stats


def ct_collator(batch):
    """The 'ct' collator of lib/datasets/collate_batch.py without the dense heatmap: inp, meta, wh, ct_cls, ct_ind and
    ct_01 exactly as the reference's ct_collator builds them, plus ct_radius int32 [B,M] from each sample's float64 wh.
    The samples' ct_hm is dropped, so it never leaves the loader worker.  img is collated only when the samples carry it:
    none of the CenterNet datasets returns it, and the reference's unconditional b['img'] stops training at the first
    batch."""
    from torch.utils.data.dataloader import default_collate
    ret = {'inp': default_collate([b['inp'] for b in batch])}
    if all('img' in b for b in batch):
        ret.update({'img': default_collate([b['img'] for b in batch])})

    meta = default_collate([b['meta'] for b in batch])
    ret.update({'meta': meta})

    batch_size = len(batch)
    ct_num = int(torch.max(meta['ct_num']))
    wh = torch.zeros([batch_size, ct_num, 2], dtype=torch.float)
    radius = torch.zeros([batch_size, ct_num], dtype=torch.int32)
    ct_cls = torch.zeros([batch_size, ct_num], dtype=torch.int64)
    ct_ind = torch.zeros([batch_size, ct_num], dtype=torch.int64)
    ct_01 = torch.zeros([batch_size, ct_num], dtype=torch.bool)
    for i in range(batch_size):
        ct_01[i, :meta['ct_num'][i]] = True

    sizes = sum([list(b['wh']) for b in batch], [])
    wh[ct_01] = torch.tensor(np.asarray(sizes, np.float64).reshape(-1, 2), dtype=torch.float)
    radius[ct_01] = torch.from_numpy(ct_radius(np.asarray(sizes, np.float64).reshape(-1, 2)))
    ct_cls[ct_01] = torch.tensor(sum([list(b['ct_cls']) for b in batch], []), dtype=torch.int64)
    ct_ind[ct_01] = torch.tensor(sum([list(b['ct_ind']) for b in batch], []), dtype=torch.int64)

    ret.update({'wh': wh, 'ct_cls': ct_cls, 'ct_ind': ct_ind, 'ct_01': ct_01.float(), 'ct_radius': radius})
    return ret


def install_ct_loss_as_reference():
    """Makes an unmodified clean-pvnet train_net.py train the CenterNet detector (task 'ct') with the fused heatmap loss.
    Call it once, before the data loaders and the trainer are built.  Two patches, both needed:
      - lib.datasets.collate_batch._collators['ct'] -> ct_collator (make_collator reads the dict at call time): the
        batch carries each object's radius instead of the stacked ct_hm;
      - lib.train.trainers.make_trainer._wrapper_factory: returns CtNetworkWrapper for cfg.task == 'ct' and calls the
        factory it replaces for every other task, so it coexists with install_vote_loss_as_reference() in either order.
    data_utils.draw_umich_gaussian is left alone: the workers still draw ct_hm, but it never leaves them.  Packages
    resolve through _dropin.reference_package, as for the other drop-ins.  Idempotent."""
    from ._dropin import chain_wrapper_factory, reference_package
    collate = reference_package("lib.datasets.collate_batch")
    collators = getattr(collate, "_collators", None)
    if collators is None:
        collators = collate._collators = {}
    collators['ct'] = ct_collator
    chain_wrapper_factory('ct', CtNetworkWrapper, "__pvb_ct_loss__")
