"""Twin of clean-pvnet's `lib/networks/dcn_v2.py:132-300` (DCNv2's deformable PSROI pooling) on the device kernels of
csrc/dcn_pool.cu, and the module `install_dcn_as_reference_module()` puts in place of `lib.networks.dcn_v2`.

    dcn_v2_pooling(input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size=1,
                   part_size=None, sample_per_part=4, trans_std=.0)
                                      the autograd Function, same positional signature as the reference's
    DCNv2Pooling(spatial_scale, pooled_size, output_dim, no_trans, ...)
    DCNPooling(..., deform_fc_dim=1024) the same, with offsets and a mask from its own offset_mask_fc

The convolution's names (dcn_v2_conv, DCNv2, DCN, from .dcn) are bound here too, so this module has all six public
names of the reference's.  fp32 CUDA tensors only; there is no CPU implementation behind them, as the reference's CPU
entry points only raise.  Only group_size 1 is supported (the reference's own assert, C == output_dim, rules the rest
out); a ROI whose batch index is outside [0, B) pools to 0 and gets no gradient.
"""
import ctypes

import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _lib
from .dcn import DCN, DCNv2, dcn_v2_conv, install_dcn_as_reference_module  # noqa: F401  (the module's other names)


def _desc(input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size,
          sample_per_part, trans_std):
    """Checks the tensors (shapes first, then device and dtype) and returns the descriptor."""
    name = "dcn_v2_pooling"
    if not isinstance(input, torch.Tensor) or input.dim() != 4:
        raise RuntimeError(f"{name}: input must be [B, C, H, W]")
    if not isinstance(rois, torch.Tensor) or rois.dim() != 2 or rois.shape[1] != 5:
        raise RuntimeError(f"{name}: rois must be [n_roi, 5], got {list(getattr(rois, 'shape', []))}")
    d = _lib.PvbDcnPoolDesc()
    d.B, d.C, d.H, d.W = (int(s) for s in input.shape)
    d.n_roi, d.output_dim, d.pooled_size = int(rois.shape[0]), int(output_dim), int(pooled_size)
    d.part_size = int(pooled_size if part_size is None else part_size)
    d.sample_per_part, d.group_size, d.no_trans = int(sample_per_part), int(group_size), int(bool(no_trans))
    d.spatial_scale, d.trans_std = float(spatial_scale), float(trans_std)
    ts = dict(input=input, rois=rois)
    if no_trans:
        d.num_classes = 1
    else:
        if not isinstance(offset, torch.Tensor) or offset.dim() != 4 or offset.shape[1] % 2 or offset.shape[1] == 0:
            raise RuntimeError(f"{name}: offset must be [n_roi, 2*num_classes, part_size, part_size], got "
                               f"{list(getattr(offset, 'shape', []))}")
        d.num_classes = int(offset.shape[1]) // 2
        want = [d.n_roi, 2 * d.num_classes, d.part_size, d.part_size]
        if list(offset.shape) != want:
            raise RuntimeError(f"{name}: offset must be {want}, got {list(offset.shape)}")
        ts["offset"] = offset
    for k, t in ts.items():
        if not t.is_cuda:
            raise RuntimeError(f"{name}: {k} must be a CUDA tensor (there is no CPU implementation)")
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name}: {k} must be float32, got {t.dtype} (the kernels are fp32 only)")
        if t.device != input.device:
            raise RuntimeError(f"{name}: {k} is on {t.device}, input on {input.device}")
    return d


def _call(entry, dev, d, *args):
    args = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.load(), entry)(ctypes.byref(d), *args,
                                                ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))


def pool_forward(input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0):
    """(output, output_count), both [n_roi, output_dim, P, P], of dcn_v2_pooling without autograd; no host sync."""
    d = _desc(input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size,
              sample_per_part, trans_std)
    shape = (d.n_roi, d.output_dim, d.pooled_size, d.pooled_size)
    out = torch.empty(shape, dtype=torch.float32, device=input.device)
    count = torch.empty(shape, dtype=torch.float32, device=input.device)
    x, r = input.contiguous(), rois.contiguous()
    t = None if no_trans else offset.contiguous()
    _call("pvb_dcn_pool_forward", input.device, d, x, r, t, out, count)
    return out, count


def pool_backward(grad_output, input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size=1,
                  part_size=None, sample_per_part=4, trans_std=.0):
    """(grad_input, grad_offset) of dcn_v2_pooling for grad_output; with no_trans grad_offset is zeros shaped like
    offset, as in the reference.  The counts are recomputed.  No host sync."""
    d = _desc(input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size,
              sample_per_part, trans_std)
    shape = [d.n_roi, d.output_dim, d.pooled_size, d.pooled_size]
    if list(grad_output.shape) != shape or grad_output.dtype != torch.float32 or grad_output.device != input.device:
        raise RuntimeError(f"dcn_v2_pooling: grad_output must be fp32 {shape} on {input.device}, got "
                           f"{grad_output.dtype} {list(grad_output.shape)} on {grad_output.device}")
    x, r, go = input.contiguous(), rois.contiguous(), grad_output.contiguous()
    t = None if no_trans else offset.contiguous()
    grad_input = torch.empty_like(x)
    grad_offset = torch.zeros_like(offset) if no_trans else torch.empty_like(t)
    _call("pvb_dcn_pool_backward", input.device, d, x, r, t, go, grad_input, None if no_trans else grad_offset)
    return grad_input, grad_offset


class _DCNv2Pooling(Function):
    @staticmethod
    def forward(ctx, input, rois, offset, spatial_scale, pooled_size, output_dim, no_trans, group_size=1,
                part_size=None, sample_per_part=4, trans_std=.0):
        ctx.spatial_scale = spatial_scale
        ctx.no_trans = int(no_trans)
        ctx.output_dim = output_dim
        ctx.group_size = group_size
        ctx.pooled_size = pooled_size
        ctx.part_size = pooled_size if part_size is None else part_size
        ctx.sample_per_part = sample_per_part
        ctx.trans_std = trans_std
        output, _ = pool_forward(input, rois, offset, spatial_scale, pooled_size, output_dim, ctx.no_trans, group_size,
                                 ctx.part_size, sample_per_part, trans_std)
        ctx.save_for_backward(input, rois, offset)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        input, rois, offset = ctx.saved_tensors
        grad_input, grad_offset = pool_backward(grad_output, input, rois, offset, ctx.spatial_scale, ctx.pooled_size,
                                                ctx.output_dim, ctx.no_trans, ctx.group_size, ctx.part_size,
                                                ctx.sample_per_part, ctx.trans_std)
        return grad_input, None, grad_offset, None, None, None, None, None, None, None, None


dcn_v2_pooling = _DCNv2Pooling.apply


class DCNv2Pooling(nn.Module):
    """lib/networks/dcn_v2.py:187-220: no parameters; forward(input, rois, offset) asserts input.shape[1] ==
    output_dim and passes an empty offset with no_trans."""

    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0):
        super(DCNv2Pooling, self).__init__()
        self.spatial_scale = spatial_scale
        self.pooled_size = pooled_size
        self.output_dim = output_dim
        self.no_trans = no_trans
        self.group_size = group_size
        self.part_size = pooled_size if part_size is None else part_size
        self.sample_per_part = sample_per_part
        self.trans_std = trans_std

    def forward(self, input, rois, offset):
        assert input.shape[1] == self.output_dim
        if self.no_trans:
            offset = input.new()
        return dcn_v2_pooling(input, rois, offset, self.spatial_scale, self.pooled_size, self.output_dim, self.no_trans,
                              self.group_size, self.part_size, self.sample_per_part, self.trans_std)


class DCNPooling(DCNv2Pooling):
    """lib/networks/dcn_v2.py:223-300: unless no_trans, pools once without offsets, runs offset_mask_fc (Linear, ReLU,
    Linear, ReLU, Linear to P*P*3, the last zero-initialised) on it, splits (o1, o2, mask) and returns the pooling with
    offset cat(o1, o2) times sigmoid(mask)."""

    def __init__(self, spatial_scale, pooled_size, output_dim, no_trans, group_size=1, part_size=None,
                 sample_per_part=4, trans_std=.0, deform_fc_dim=1024):
        super(DCNPooling, self).__init__(spatial_scale, pooled_size, output_dim, no_trans, group_size, part_size,
                                         sample_per_part, trans_std)
        self.deform_fc_dim = deform_fc_dim
        if not no_trans:
            self.offset_mask_fc = nn.Sequential(
                nn.Linear(self.pooled_size * self.pooled_size * self.output_dim, self.deform_fc_dim),
                nn.ReLU(inplace=True),
                nn.Linear(self.deform_fc_dim, self.deform_fc_dim),
                nn.ReLU(inplace=True),
                nn.Linear(self.deform_fc_dim, self.pooled_size * self.pooled_size * 3))
            self.offset_mask_fc[4].weight.data.zero_()
            self.offset_mask_fc[4].bias.data.zero_()

    def forward(self, input, rois):
        offset = input.new()
        args = (self.spatial_scale, self.pooled_size, self.output_dim)
        rest = (self.group_size, self.part_size, self.sample_per_part, self.trans_std)
        if not self.no_trans:
            n = rois.shape[0]
            roi = dcn_v2_pooling(input, rois, offset, *args, True, *rest)
            offset_mask = self.offset_mask_fc(roi.view(n, -1))
            offset_mask = offset_mask.view(n, 3, self.pooled_size, self.pooled_size)
            o1, o2, mask = torch.chunk(offset_mask, 3, dim=1)
            offset = torch.cat((o1, o2), dim=1)
            mask = torch.sigmoid(mask)
            return dcn_v2_pooling(input, rois, offset, *args, self.no_trans, *rest) * mask
        return dcn_v2_pooling(input, rois, offset, *args, self.no_trans, *rest)
