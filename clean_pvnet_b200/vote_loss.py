"""PVNet's vote loss computed from the mask and the keypoints on the device, so training never builds or ships the dense
target field (DESIGN.md section 8e; the kernels are csrc/loss.cu):

    vote_target_batch(mask, kpt_2d)        pvnet_data_utils.compute_vertex (lib/utils/pvnet/pvnet_data_utils.py:30-44)
                                           for B images -> float32 [B,2K,H,W], bit for bit
    vote_loss(pred, mask, kpt_2d)          the trainer's vote loss (lib/train/trainers/pvnet.py:25-27) with that target,
                                           an autograd Function; its gradient for pred is autograd's bit for bit
    NetworkWrapper(net)                    twin of lib/train/trainers/pvnet.py's NetworkWrapper on vote_loss
    install_vote_loss_as_reference()       the zero-edit drop-in for clean-pvnet's datasets and trainer

The drop-in's datasets hand the trainer the keypoints instead of the field.  The patched compute_vertex returns them as
float64 [1,K,2]; the dataset's own `.transpose(2, 0, 1)` makes that [2,1,K], and default_collate and DataParallel's scatter
make batch['vertex'] float64 [B,2,1,K].  float64 marks the compact form: the real field is float32.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .metrics import _MASK_DTYPES
from .nn import _call, _workspace


def _mask_args(mask):
    """(pvb_mask_dtype, int64[3] strides) of a [B,H,W] integer or bool CUDA tensor; raises RuntimeError otherwise."""
    if not (isinstance(mask, torch.Tensor) and mask.is_cuda):
        raise RuntimeError("mask must be a CUDA tensor")
    if mask.dim() != 3:
        raise RuntimeError(f"mask must be [B,H,W], got {list(mask.shape)}")
    if mask.dtype not in _MASK_DTYPES:
        raise RuntimeError(f"mask must be a bool, uint8 or signed integer tensor, got {mask.dtype}")
    return _MASK_DTYPES[mask.dtype], (ctypes.c_int64 * 3)(*mask.stride())


def _keypoints(kpt_2d, mask):
    """kpt_2d [B,K,2] (tensor or array, float32 or float64) as contiguous float64 on the mask's device; float32 is
    promoted exactly, as numpy promotes it against the integer pixel coordinates."""
    k = torch.as_tensor(kpt_2d)
    if k.dtype not in (torch.float32, torch.float64):
        raise RuntimeError(f"kpt_2d must be float32 or float64, got {k.dtype}")
    if k.dim() != 3 or k.shape[2] != 2 or k.shape[0] != mask.shape[0]:
        raise RuntimeError(f"kpt_2d must be [B,K,2] with B = {mask.shape[0]}, got {list(k.shape)}")
    if k.shape[1] < 1:
        raise RuntimeError("kpt_2d must hold at least one keypoint")
    return k.to(device=mask.device, dtype=torch.float64).contiguous()


def vote_target_batch(mask, kpt_2d):
    """compute_vertex (lib/utils/pvnet/pvnet_data_utils.py:30-44) for B images at once, bit for bit: mask [B,H,W] CUDA
    tensor of bool / uint8 / int8 / int16 / int32 / int64 (any strides), kpt_2d [B,K,2] float32 or float64.  Returns
    float32 [B,2K,H,W] on the mask's device (the dataset's `compute_vertex(...).transpose(2, 0, 1)`, batched): channel 2k
    is the x component of keypoint k and 2k+1 its y; only mask == 1 pixels are non-zero."""
    dtype, ms = _mask_args(mask)
    kpt = _keypoints(kpt_2d, mask)
    B, H, W = (int(s) for s in mask.shape)
    K = int(kpt.shape[1])
    out = torch.empty((B, 2 * K, H, W), dtype=torch.float32, device=mask.device)
    _call("pvb_vote_target", mask.device, ctypes.c_void_p(mask.data_ptr() or None), dtype, ms, kpt, out, B, H, W, K)
    return out


def _check_pred(pred, mask, K):
    if not (isinstance(pred, torch.Tensor) and pred.is_cuda):
        raise RuntimeError("pred must be a CUDA tensor")
    if pred.dtype != torch.float32:
        raise RuntimeError(f"pred must be float32 (the reference trains in fp32), got {pred.dtype}")
    B, H, W = mask.shape
    if tuple(pred.shape) != (B, 2 * K, H, W):
        raise RuntimeError(f"pred must be [B,2K,H,W] = {[B, 2 * K, H, W]}, got {list(pred.shape)}")
    if pred.device != mask.device:
        raise RuntimeError(f"pred and mask must be on one device, got {pred.device} and {mask.device}")


class _VoteLoss(torch.autograd.Function):
    """smooth_l1(pred * w, tgt * w, 'sum') / w.sum() / 2K with tgt = compute_vertex(mask, kpt), w = float(mask)."""

    @staticmethod
    def forward(ctx, pred, mask, kpt):
        dtype, ms = _mask_args(mask)
        dev = pred.device
        B, H, W = (int(s) for s in mask.shape)
        K = int(kpt.shape[1])
        ps = (ctypes.c_int64 * 4)(*pred.stride())
        loss = torch.empty((), dtype=torch.float32, device=dev)
        nbytes = _lib.load().pvb_vote_loss_workspace_bytes(B, H, W)
        ws = _workspace(nbytes, dev)                       # holds the fp32 weight sum for backward
        _call("pvb_vote_loss_forward", dev, ctypes.c_void_p(pred.data_ptr() or None), ps,
              ctypes.c_void_p(mask.data_ptr() or None), dtype, ms, kpt, loss, B, H, W, K, ws, nbytes)
        ctx.save_for_backward(pred, mask, kpt)
        ctx.ws, ctx.nbytes = ws, nbytes
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        pred, mask, kpt = ctx.saved_tensors
        dtype, ms = _mask_args(mask)
        dev = pred.device
        B, H, W = (int(s) for s in mask.shape)
        K = int(kpt.shape[1])
        ps = (ctypes.c_int64 * 4)(*pred.stride())
        g = grad_loss.to(device=dev, dtype=torch.float32).contiguous()
        grad = torch.empty((B, 2 * K, H, W), dtype=torch.float32, device=dev)
        _call("pvb_vote_loss_backward", dev, ctypes.c_void_p(pred.data_ptr() or None), ps,
              ctypes.c_void_p(mask.data_ptr() or None), dtype, ms, kpt, g, grad, B, H, W, K, ctx.ws, ctx.nbytes)
        return grad, None, None


def vote_loss(pred, mask, kpt_2d):
    """The vote loss of clean-pvnet's trainer (lib/train/trainers/pvnet.py:25-27),
        w = mask[:, None].float();  smooth_l1_loss(pred * w, vertex * w, reduction='sum') / w.sum() / vertex.size(1)
    with vertex = compute_vertex(mask, kpt_2d) computed per pixel on the device and never stored.  pred: float32
    [B,2K,H,W] CUDA tensor, any strides (fp16 / bf16 are refused); mask: [B,H,W] as in vote_target_batch; kpt_2d: [B,K,2]
    float32 or float64 (a CUDA tensor avoids a host copy).  Returns a 0-dim float32 tensor with a gradient for pred only;
    neither pass synchronises with the host, and both run on the current stream of pred's device, so the function works
    in DataParallel replicas.  The loss is reproducible bit for bit and within one fp32 ulp of the same chain on a float64
    sum of the terms; the gradient equals autograd's of the reference expression bit for bit."""
    _mask_args(mask)
    kpt = _keypoints(kpt_2d, mask)
    _check_pred(pred, mask, int(kpt.shape[1]))
    return _VoteLoss.apply(pred, mask, kpt)


def compact_vertex(mask, kpt_2d):
    """What install_vote_loss_as_reference() makes pvnet_data_utils.compute_vertex return: the keypoints as float64
    [1,K,2], which the dataset's `.transpose(2, 0, 1)` turns into [2,1,K].  `mask` is unused (the trainer reads
    batch['mask'])."""
    return np.asarray(kpt_2d, dtype=np.float64).reshape(1, -1, 2)


def keypoints_from_compact(vertex):
    """batch['vertex'] in the compact form, float64 [B,2,1,K], -> the keypoints float64 [B,K,2].  Raises RuntimeError on
    anything else, e.g. a dense float32 [B,2K,H,W] field from a dataset whose compute_vertex was not patched."""
    if not isinstance(vertex, torch.Tensor) or vertex.dtype != torch.float64 or vertex.dim() != 4 or \
            vertex.shape[1] != 2 or vertex.shape[2] != 1:
        desc = f"{vertex.dtype} {list(vertex.shape)}" if isinstance(vertex, torch.Tensor) else type(vertex).__name__
        raise RuntimeError(
            f"batch['vertex'] must be the compact keypoint form, float64 [B,2,1,K], got {desc}: call "
            "clean_pvnet_b200.install_vote_loss_as_reference() before the datasets are built, so that "
            "pvnet_data_utils.compute_vertex returns the keypoints instead of the dense field")
    return vertex[:, :, 0, :].transpose(1, 2)


class NetworkWrapper(torch.nn.Module):
    """Twin of clean-pvnet's lib/train/trainers/pvnet.py NetworkWrapper: the same 'pose_test' branch, the same
    nn.CrossEntropyLoss segmentation loss and the same scalar_stats keys (vote_loss, seg_loss, loss), with the vote loss
    computed by vote_loss from batch['mask'] and the compact batch['vertex'] (see keypoints_from_compact)."""

    def __init__(self, net):
        super().__init__()
        self.net = net
        self.seg_crit = torch.nn.CrossEntropyLoss()

    def forward(self, batch):
        output = self.net(batch['inp'])

        scalar_stats = {}
        loss = 0

        if 'pose_test' in batch['meta'].keys():
            loss = torch.tensor(0).to(batch['inp'].device)
            return output, loss, {}, {}

        kpt_2d = keypoints_from_compact(batch['vertex'])
        v_loss = vote_loss(output['vertex'], batch['mask'], kpt_2d)
        scalar_stats.update({'vote_loss': v_loss})
        loss += v_loss

        mask = batch['mask'].long()
        seg_loss = self.seg_crit(output['seg'], mask)
        scalar_stats.update({'seg_loss': seg_loss})
        loss += seg_loss

        scalar_stats.update({'loss': loss})
        image_stats = {}

        return output, loss, scalar_stats, image_stats


def install_vote_loss_as_reference():
    """Makes an unmodified clean-pvnet train_net.py train with the fused vote loss.  Call it once, before the datasets
    and the trainer are built (e.g. at the top of train_net.py).  Two patches, both needed:
      - lib.utils.pvnet.pvnet_data_utils.compute_vertex -> compact_vertex: the datasets (lib/datasets/{linemod,custom}/
        pvnet.py:53, tless_train/pvnet.py:117) look it up through the module at call time, so they emit the keypoints;
      - lib.train.trainers.make_trainer._wrapper_factory: make_trainer loads the trainer file by path (make_trainer.py:6-10),
        so replacing a sys.modules entry would not reach it; the patched factory returns NetworkWrapper for
        cfg.task == 'pvnet' and calls the original for every other task.
    Packages resolve through _dropin.reference_package, as for the other drop-ins.  Idempotent."""
    from ._dropin import reference_package
    data_utils = reference_package("lib.utils.pvnet.pvnet_data_utils")
    data_utils.compute_vertex = compact_vertex
    trainer = reference_package("lib.train.trainers.make_trainer")
    original = getattr(trainer, "_wrapper_factory", None)
    if getattr(original, "__pvb_vote_loss__", False):
        return
    if original is None:
        def original(cfg, network):
            raise RuntimeError(f"no trainer for task {cfg.task!r}: lib.train.trainers.make_trainer is not importable")

    def _wrapper_factory(cfg, network):
        if cfg.task == 'pvnet':
            return NetworkWrapper(network)
        return original(cfg, network)

    _wrapper_factory.__pvb_vote_loss__ = True
    trainer._wrapper_factory = _wrapper_factory
