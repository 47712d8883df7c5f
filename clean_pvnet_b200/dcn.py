"""Twin of clean-pvnet's `lib/networks/dcn_v2.py:16-128` (the modulated deformable convolution, DCNv2, of the DLA-34
CenterNet detector, lib/networks/ct/dla_dcn.py) on the device kernels of csrc/dcn.cu.

    dcn_v2_conv(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups)
                                      the autograd Function, same positional signature as the reference's
    DCNv2(in, out, kernel_size, stride, padding, dilation=1, deformable_groups=1)
    DCN(...)                          the same module, with its own conv_offset_mask (what dla_dcn.py builds)
    install_dcn_as_reference_module() `from lib.networks.dcn_v2 import DCN` binds these names (and the pooling's, from
                                      dcn_pool.py, the twin of the rest of lib/networks/dcn_v2.py)

The reference's extension, lib/csrc/dcn_v2, is written against THC and does not build on current torch, so
`import lib.networks.ct.dla_dcn` fails there; with install_dcn_as_reference_module() called first it imports and runs
on these kernels, and net_utils.load_network loads a trained detector unchanged (same parameter names).  CUDA
tensors only; there is no CPU implementation behind them.

The compute dtype is the input's.  An fp32 input needs every tensor fp32 and runs the FP32-FFMA kernels.  An fp16 or
bf16 input (what the DLA-34's convolutions emit under torch.autocast, or a .half() / .bfloat16() model) casts offset,
mask, weight and bias to its dtype, round to nearest, and runs the tensor-core forward (DESIGN.md section 8n); the
backward is the fp32 one on exact up-casts of those operands, and each gradient comes back in its tensor's dtype, so an
fp32 parameter gets an fp32 gradient.  The dispatch does not look at the autocast state.

The layout is the input's.  An fp16 / bf16 input that is channels_last and not NCHW-contiguous (what a model moved to
torch.channels_last feeds its DCN layers) runs the NHWC twin of the tensor-core forward (DESIGN.md section 8o) with no
copy of the input; offset and mask are brought to channels_last (a no-op for the ones DCN builds from a channels_last
input), and the output is channels_last with the values the NCHW call returns, bit for bit.  Every other input (fp32 in
any layout, NCHW, or contiguous in both layouts) is made NCHW-contiguous and returns NCHW, as before.  The backward is
the same in both layouts: NCHW fp32, so a channels_last call's gradients equal the NCHW call's.

TF32 follows torch's matmul switch, read on every call as torch.matmul reads it (tf32_enabled):
torch.backends.cuda.matmul.fp32_precision == "tf32", which torch.set_float32_matmul_precision("high" / "medium"),
torch.backends.cuda.matmul.allow_tf32 = True and torch.backends.fp32_precision = "tf32" all set.  When it is on, an fp32
forward runs pvb_dcn_forward_tf32 and every backward (fp32, or the one on the up-cast operands of an fp16 / bf16
forward) runs pvb_dcn_backward_tf32: the same columns, with each product's operands rounded once to TF32 and summed in
fp32 on the tensor cores (DESIGN.md section 8p).  The fp16 / bf16 forward is the same with the switch on or off.  When
it is off (torch's default), nothing here differs from the FP32-FFMA path.  torch.backends.cudnn.allow_tf32 is not
followed: DCN's product is a GEMM, and it defaults to True.
"""
import ctypes
import math
import sys

import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from . import _lib

# grad_cols, the backward's only stored column matrix ([chunk, C*kh*kw, Ho*Wo] fp32), is planned in image chunks of at
# most this many bytes (one image always fits); the other outputs do not depend on the chunking.
MAX_COLUMN_BYTES = 1 << 28

# the half-precision compute dtypes and their code in pvb_dcn_forward_half
HALF = {torch.float16: _lib.PVB_DCN_F16, torch.bfloat16: _lib.PVB_DCN_BF16}


def _desc(input, weight, stride, padding, dilation, deformable_groups):
    d = _lib.PvbDcnDesc()
    d.B, d.C, d.H, d.W = (int(s) for s in input.shape)
    d.C_out, _, d.kh, d.kw = (int(s) for s in weight.shape)
    d.stride_h, d.stride_w = _pair(stride)
    d.pad_h, d.pad_w = _pair(padding)
    d.dilation_h, d.dilation_w = _pair(dilation)
    d.deformable_groups = int(deformable_groups)
    return d


def _out_hw(d):
    ho = (d.H + 2 * d.pad_h - (d.dilation_h * (d.kh - 1) + 1)) // d.stride_h + 1
    wo = (d.W + 2 * d.pad_w - (d.dilation_w * (d.kw - 1) + 1)) // d.stride_w + 1
    return ho, wo


def _operands(input, offset, mask, weight, bias):
    """(offset, mask, weight, bias) in the compute dtype: cast to an fp16 / bf16 input's dtype (round to nearest) from
    fp32, fp16 or bf16; left as they are for any other input, which _check then holds to fp32."""
    if not isinstance(input, torch.Tensor) or input.dtype not in HALF:
        return offset, mask, weight, bias
    ts = dict(offset=offset, mask=mask, weight=weight, bias=bias)
    for name, t in ts.items():
        if isinstance(t, torch.Tensor) and t.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            raise RuntimeError(f"dcn_v2_conv: {name} must be float32, float16 or bfloat16 with a {input.dtype} input, "
                               f"got {t.dtype}")
    return tuple(t.to(input.dtype) if isinstance(t, torch.Tensor) else t for t in ts.values())


def _check(input, offset, mask, weight, bias, d):
    ts = dict(input=input, offset=offset, mask=mask, weight=weight, bias=bias)
    for name, t in ts.items():
        if not isinstance(t, torch.Tensor):
            raise RuntimeError(f"dcn_v2_conv: {name} must be a CUDA tensor")
    want = input.dtype if input.dtype in HALF else torch.float32
    for name, t in ts.items():
        if t.dtype != want:
            raise RuntimeError(f"dcn_v2_conv: {name} must be {want}, got {t.dtype} (the kernels take float32 throughout, "
                               f"or a float16 / bfloat16 input with the other tensors cast to its dtype)")
    for name, t in ts.items():
        if not t.is_cuda:
            raise RuntimeError(f"dcn_v2_conv: {name} must be a CUDA tensor")
        if t.device != input.device:
            raise RuntimeError(f"dcn_v2_conv: {name} is on {t.device}, input on {input.device}")
    if input.dim() != 4 or weight.dim() != 4 or weight.shape[1] != input.shape[1]:
        raise RuntimeError(f"dcn_v2_conv: input [B,C,H,W] and weight [C_out,C,kh,kw] do not match: "
                           f"{list(input.shape)} and {list(weight.shape)}")
    ho, wo = _out_hw(d)
    t, dg = d.kh * d.kw, d.deformable_groups
    want = dict(offset=[d.B, dg * 2 * t, ho, wo], mask=[d.B, dg * t, ho, wo], bias=[d.C_out])
    for name, shape in want.items():
        if list(ts[name].shape) != shape:
            raise RuntimeError(f"dcn_v2_conv: {name} must be {shape}, got {list(ts[name].shape)}")


def _nhwc(input):
    """Whether a forward runs the NHWC kernel: an fp16 / bf16 input that is channels_last-contiguous and not
    NCHW-contiguous.  An empty batch is contiguous in both layouts whatever its strides, so there the strides decide."""
    if input.dtype not in HALF:
        return False
    B, C, H, W = input.shape
    if B == 0:
        return C > 1 and H * W > 1 and input.stride() == (H * W * C, 1, W * C, C)
    return input.is_contiguous(memory_format=torch.channels_last) and not input.is_contiguous()


def tf32_enabled():
    """Whether fp32 products may round their operands to TF32: torch's matmul flag.  matmul.fp32_precision is readable
    whichever API set it ("tf32" on; "none", the default, or "ieee" off); reading allow_tf32 or
    get_float32_matmul_precision() raises once the new API is in use, so they are read only on a torch without it."""
    matmul = torch.backends.cuda.matmul
    try:
        precision = matmul.fp32_precision
    except AttributeError:                                   # torch < 2.9
        return bool(matmul.allow_tf32)
    return precision == "tf32"


def _call(entry, dev, *args):
    args = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.load(), entry)(*args, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))


def dcn_forward(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups):
    """The forward of dcn_v2_conv without autograd: output [B,C_out,Ho,Wo] in the compute dtype on input's device,
    channels_last when the input takes the NHWC path (see _nhwc); no host sync."""
    offset, mask, weight, bias = _operands(input, offset, mask, weight, bias)
    d = _desc(input, weight, stride, padding, dilation, deformable_groups)
    _check(input, offset, mask, weight, bias, d)
    ho, wo = _out_hw(d)
    nhwc = _nhwc(input)
    layout = torch.channels_last if nhwc else torch.contiguous_format
    out = torch.empty((d.B, d.C_out, ho, wo), dtype=input.dtype, device=input.device, memory_format=layout)
    if d.B and input.dtype == torch.float32 and tf32_enabled():
        x, off, m, b = (t.contiguous() for t in (input, offset, mask, bias))
        w = weight.permute(0, 2, 3, 1).contiguous()          # tap-major [C_out, kh, kw, C], as the kernel reads it
        _call("pvb_dcn_forward_tf32", input.device, ctypes.byref(d), x, off, m, w, b, out)
    elif d.B and input.dtype == torch.float32:
        c = [t.contiguous() for t in (input, offset, mask, weight, bias)]
        _call("pvb_dcn_forward", input.device, ctypes.byref(d), *c, out)
    elif d.B and nhwc:
        off, m = (t.contiguous(memory_format=torch.channels_last) for t in (offset, mask))
        w = weight.permute(0, 2, 3, 1).contiguous()          # tap-major [C_out, kh, kw, C], as the kernel reads it
        _call("pvb_dcn_forward_half_nhwc", input.device, ctypes.byref(d), HALF[input.dtype], input, off, m, w,
              bias.contiguous(), out)
    elif d.B:
        x, off, m, b = (t.contiguous() for t in (input, offset, mask, bias))
        w = weight.permute(0, 2, 3, 1).contiguous()          # tap-major [C_out, kh, kw, C], as the kernel reads it
        _call("pvb_dcn_forward_half", input.device, ctypes.byref(d), HALF[input.dtype], x, off, m, w, b, out)
    return out


def dcn_backward(input, offset, mask, weight, bias, grad_output, stride, padding, dilation, deformable_groups,
                 max_column_bytes=None):
    """(grad_input, grad_offset, grad_mask, grad_weight, grad_bias) of dcn_v2_conv for grad_output; no host sync.
    grad_cols goes through a workspace of at most max_column_bytes (default MAX_COLUMN_BYTES) per image chunk.  Runs
    pvb_dcn_backward_tf32 when tf32_enabled() holds at the call, pvb_dcn_backward otherwise."""
    d = _desc(input, weight, stride, padding, dilation, deformable_groups)
    _check(input, offset, mask, weight, bias, d)
    ho, wo = _out_hw(d)
    if list(grad_output.shape) != [d.B, d.C_out, ho, wo] or grad_output.dtype != torch.float32 or not grad_output.is_cuda:
        raise RuntimeError(f"dcn_v2_conv: grad_output must be fp32 CUDA [{d.B},{d.C_out},{ho},{wo}], got "
                           f"{grad_output.dtype} {list(grad_output.shape)}")
    c = [t.contiguous() for t in (input, offset, mask, weight, grad_output)]
    grads = [torch.empty_like(t) for t in (c[0], c[1], c[2], c[3])] + [torch.empty_like(bias)]
    if d.B == 0:
        for g in grads[3:]:
            g.zero_()
        return tuple(grads)
    budget = MAX_COLUMN_BYTES if max_column_bytes is None else int(max_column_bytes)
    per_image = d.C * d.kh * d.kw * ho * wo * 4
    chunk = max(1, min(d.B, budget // max(per_image, 1)))
    lib = _lib.load()
    nbytes = lib.pvb_dcn_backward_workspace_bytes(ctypes.byref(d), chunk)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=input.device)
    entry = "pvb_dcn_backward_tf32" if tf32_enabled() else "pvb_dcn_backward"
    _call(entry, input.device, ctypes.byref(d), *c, *grads, chunk, ws, nbytes)
    return tuple(grads)


class _DCNv2(Function):
    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups):
        ctx.stride = _pair(stride)
        ctx.padding = _pair(padding)
        ctx.dilation = _pair(dilation)
        ctx.kernel_size = _pair(weight.shape[2:4])
        ctx.deformable_groups = deformable_groups
        ops = _operands(input, offset, mask, weight, bias)
        output = dcn_forward(input, *ops, ctx.stride, ctx.padding, ctx.dilation, deformable_groups)
        ctx.dtypes = tuple(t.dtype for t in (input, offset, mask, weight, bias))
        ctx.save_for_backward(input, *ops)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        input, offset, mask, weight, bias = ctx.saved_tensors
        grad_output = grad_output.contiguous()
        if input.dtype != torch.float32:     # the fp32 backward on the operands the forward used, up-cast exactly
            input, offset, mask, weight, bias, grad_output = (
                t.float() for t in (input, offset, mask, weight, bias, grad_output))
        grads = dcn_backward(input, offset, mask, weight, bias, grad_output, ctx.stride, ctx.padding, ctx.dilation,
                             ctx.deformable_groups)
        return tuple(g.to(dt) for g, dt in zip(grads, ctx.dtypes)) + (None, None, None, None)


dcn_v2_conv = _DCNv2.apply


class DCNv2(nn.Module):
    """lib/networks/dcn_v2.py:57-94: weight [out, in, kh, kw] ~ U(-1/sqrt(in*kh*kw), +), bias zero."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1):
        super(DCNv2, self).__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride = _pair(stride)
        self.padding = _pair(padding)
        self.dilation = _pair(dilation)
        self.deformable_groups = deformable_groups

        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels, *self.kernel_size))
        self.bias = nn.Parameter(torch.Tensor(out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        n = self.in_channels
        for k in self.kernel_size:
            n *= k
        stdv = 1. / math.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)
        self.bias.data.zero_()

    def forward(self, input, offset, mask):
        assert 2 * self.deformable_groups * self.kernel_size[0] * self.kernel_size[1] == offset.shape[1]
        assert self.deformable_groups * self.kernel_size[0] * self.kernel_size[1] == mask.shape[1]
        return dcn_v2_conv(input, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups)


class DCN(DCNv2):
    """lib/networks/dcn_v2.py:97-128: DCNv2 whose offsets and mask come from its own conv_offset_mask (zero-initialised),
    split as (o1, o2, mask) thirds, offset = cat(o1, o2), mask = sigmoid(mask)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1):
        super(DCN, self).__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, deformable_groups)

        channels_ = self.deformable_groups * 3 * self.kernel_size[0] * self.kernel_size[1]
        self.conv_offset_mask = nn.Conv2d(self.in_channels, channels_, kernel_size=self.kernel_size,
                                          stride=self.stride, padding=self.padding, bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()

    def forward(self, input):
        out = self.conv_offset_mask(input)
        o1, o2, mask = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        mask = torch.sigmoid(mask)
        return dcn_v2_conv(input, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups)


def install_dcn_as_reference_module():
    """Makes `lib.networks.dcn_v2` (imported by lib/networks/ct/dla_dcn.py:16 and by lib/csrc/dcn_v2/test.py) bind this
    package's twin of the whole module, clean_pvnet_b200.dcn_pool: the convolution (dcn_v2_conv, DCNv2, DCN) and the
    deformable PSROI pooling (dcn_v2_pooling, DCNv2Pooling, DCNPooling).  The detector then imports and runs without
    the THC extension `lib.csrc.dcn_v2._ext` ever being built or imported.  Only the leaf `lib.networks.dcn_v2` is
    replaced; `lib` and `lib.networks` stay the real packages whenever they import.

    Call it BEFORE anything imports `lib.networks.ct*` (for the cascade: before install_crop_as_reference()).  Unlike
    the other drop-ins it cannot be installed afterwards: without it that import fails on the extension.  Idempotent."""
    from ._dropin import reference_package
    from . import dcn_pool
    parent = reference_package("lib.networks")
    sys.modules["lib.networks.dcn_v2"] = dcn_pool
    parent.dcn_v2 = dcn_pool
    return dcn_pool
