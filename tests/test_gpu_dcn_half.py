"""GPU tests of the half-precision DCNv2 forward (pvb_dcn_forward_half, csrc/dcn.cu; DESIGN.md section 8n) and of the
fp16 / bf16 dispatch of dcn_v2_conv: the columns against the reference's im2col (oracle/_ref/libdcn_ref.so) bit for bit,
the product within the bound DESIGN.md states, the backward against the fp32 one on the up-cast operands, and a
DeformConv-shaped block of the DLA-34 under torch.autocast with a GradScaler."""
import numpy as np
import pytest
import torch
from torch import nn

import dcn_cases as dc
import dcn_oracle as do
from test_gpu_dcn import DETECTOR_UNIQUE, DEV, U, gpu, ref_cols

pytestmark = pytest.mark.gpu
DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}      # unit roundoff of the output's rounding
C_BOUND = 3      # DESIGN.md section 8n: |out - E| <= C_BOUND * K * u32 * (|b| + sum |W| |col|) + u_dtype * |E|
DT_IDS = list(DTYPES)


def lowp(arrays, dt):
    return [t.to(dt) for t in gpu(*arrays)]


def fwd(pvb, c, x, off, m, w, b):
    return pvb.dcn.dcn_forward(x, off, m, w, b, c.stride, c.pad, c.dil, c.dg)


IDENTITY_CASES = [(c, "edges") for c in dc.SWEEP] + [(c, "random") for c in dc.SWEEP] + \
                 [(c, "edges") for c in DETECTOR_UNIQUE]


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case,offsets", IDENTITY_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else v)
def test_identity_weight_returns_the_rounded_reference_columns_bit_for_bit(pvb, case, offsets, dt):
    """W = I, bias 0: the output is to(dtype) of the reference im2col run on the up-cast inputs, exactly, at every
    edge of the bilinear domain, NaN / +-inf offsets (small sweep cases) and every detector shape."""
    dt = DTYPES[dt]
    x, off, m, _, _ = dc.make_inputs(case, seed=21, offsets=offsets, nonfinite=case.H * case.W < 1000)
    wid, bid = dc.identity_weight(case)
    x, off, m, wid, bid = lowp((x, off, m, wid, bid), dt)
    ours = fwd(pvb, case, x, off, m, wid, bid)
    assert ours.dtype == dt
    want = ref_cols(case, x.float(), off.float(), m.float()).to(dt)
    torch.cuda.synchronize()
    ours = ours.reshape(case.B, wid.shape[0], -1)
    assert torch.equal(ours, want), float((ours.float() - want.float()).abs().max())


FWD_CASES = [(c, 1) for c in dc.SWEEP] + [(c._replace(B=8), 8) for c in dc.SWEEP[:4]] + \
            [(c, 1) for c in DETECTOR_UNIQUE if c.H * c.W <= 92 * 68] + [(dc.DETECTOR["512x512"][0]._replace(B=8), 8)]


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case,B", FWD_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else f"B{v}")
def test_forward_with_real_weights_is_within_the_tensor_core_bound(pvb, case, B, dt):
    """E = fp64(b_lp + W_lp col_lp) on the rounded operands; ours and a half-precision torch.matmul of the same rounded
    columns (bias as one more column, so the output is rounded once) both meet the bound."""
    dt = DTYPES[dt]
    x, off, m, w, b = lowp(dc.make_inputs(case, seed=3, offsets="random"), dt)
    ours = fwd(pvb, case, x, off, m, w, b).reshape(case.B, case.Co, -1).double()
    cols = ref_cols(case, x.float(), off.float(), m.float()).to(dt)
    W2 = w.reshape(case.Co, -1)
    exact = b.double()[None, :, None] + torch.matmul(W2.double(), cols.double())
    absb = b.double().abs()[None, :, None] + torch.matmul(W2.double().abs(), cols.double().abs())
    K = case.C * case.kh * case.kw
    bound = C_BOUND * K * U * absb + UNIT[dt] * exact.abs()
    prev = (torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction,
            torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction)
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    try:
        ones = torch.ones((case.B, 1, cols.shape[2]), dtype=dt, device=DEV)
        theirs = torch.matmul(torch.cat([W2, b[:, None]], 1), torch.cat([cols, ones], 1)).double()
    finally:
        (torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction,
         torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction) = prev
    assert bool(((ours - exact).abs() <= bound).all()), float(((ours - exact).abs() / bound.clamp_min(1e-300)).max())
    assert bool(((theirs - exact).abs() <= bound).all())


@pytest.mark.parametrize("dt", DT_IDS)
def test_overflow_is_inf_and_an_empty_batch_is_a_no_op(pvb, dt):
    dt = DTYPES[dt]
    case = dc.SWEEP[8]
    x, off, m, w, b = lowp(dc.make_inputs(case, seed=4, offsets="zero"), dt)
    big = torch.finfo(dt).max
    out = fwd(pvb, case, torch.full_like(x, 1.0), off, torch.ones_like(m), torch.full_like(w, big / 4),
              torch.zeros_like(b))
    out_neg = fwd(pvb, case, torch.full_like(x, 1.0), off, torch.ones_like(m), torch.full_like(w, -big / 4),
                  torch.zeros_like(b))
    inner = out[:, :, 1:-1, 1:-1]                     # every tap in the image: 9 * 17 * max/4 overflows
    assert bool(torch.isposinf(inner).all()) and bool(torch.isneginf(out_neg[:, :, 1:-1, 1:-1]).all())
    e = case._replace(B=0)
    y = fwd(pvb, e, x[:0], off[:0], m[:0], w, b)
    assert y.shape == (0, case.Co, *dc.out_hw(case)) and y.dtype == dt


BWD_CASES = [(c, "random") for c in dc.SWEEP] + [(c, "edges") for c in dc.SWEEP[:5]]


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case,offsets", BWD_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else v)
def test_backward_is_the_fp32_backward_on_the_up_cast_operands(pvb, case, offsets, dt):
    """grad_offset / grad_mask / grad_weight / grad_bias equal dcn_backward on the up-cast rounded operands, cast to
    each tensor's dtype (fp32 parameters get fp32 gradients); grad_input (float atomics) meets the fp32 backward's
    bound against the fp64 restatement, plus its own rounding to the dtype."""
    dt = DTYPES[dt]
    arrs = dc.make_inputs(case, seed=9, offsets=offsets)
    x, off, m = lowp(arrs[:3], dt)
    w, b = gpu(*arrs[3:])                                     # fp32 parameters, as in a module under autocast
    Ho, Wo = dc.out_hw(case)
    go = torch.randn((case.B, case.Co, Ho, Wo), device=DEV).to(dt)
    ts = [t.clone().requires_grad_() for t in (x, off, m, w, b)]
    y = pvb.dcn_v2_conv(*ts, case.stride, case.pad, case.dil, case.dg)
    assert y.dtype == dt
    got = torch.autograd.grad(y, ts, go)
    up = [t.float() for t in (x, off, m, w.to(dt), b.to(dt), go)]
    want = pvb.dcn.dcn_backward(*up, case.stride, case.pad, case.dil, case.dg)
    names = ["grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"]
    for name, g, wnt, t in zip(names, got, want, ts):
        assert g.dtype == t.dtype, name
        if name != "grad_input":
            assert torch.equal(g, wnt.to(t.dtype)), name
    ref = do.backward(*[t.cpu().numpy() for t in up], case.stride, case.pad, case.dil, case.dg)
    n = case.Co + 8 + ref["grad_input_terms"]
    gi = got[0].double().cpu().numpy()
    # the fp32 bound, then the rounding to the dtype: relative above its normal range, half its subnormal spacing below
    err32 = n * U * ref["grad_input_abs"] * 1.01
    tiny = torch.finfo(dt).smallest_normal * UNIT[dt]
    bound = (1 + UNIT[dt]) * err32 + UNIT[dt] * np.abs(ref["grad_input"]) + tiny + 1e-30
    assert (np.abs(gi - ref["grad_input"]) <= bound).all()


class DeformConvBlock(nn.Module):
    """The shape of lib/networks/ct/dla_dcn.py's DeformConv: DCN 3x3 -> BatchNorm -> ReLU."""

    def __init__(self, pvb, chi, cho):
        super().__init__()
        self.conv = pvb.DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)
        self.actf = nn.Sequential(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))

    def forward(self, x):
        return self.actf(self.conv(x))


def _block(pvb, chi=32, cho=24):
    torch.manual_seed(0)
    net = DeformConvBlock(pvb, chi, cho).to(DEV)
    with torch.no_grad():
        net.conv.conv_offset_mask.weight.normal_(0, 0.05)
        net.conv.conv_offset_mask.bias.normal_(0, 0.5)
        net.conv.bias.normal_()
    return net


@pytest.mark.parametrize("dt", DT_IDS)
def test_deform_conv_block_under_autocast(pvb, dt):
    """The input a DeformConv gets from the autocast convolutions before it is half precision: the block keeps its
    dtype, the DCN equals an explicit call with cast operands bit for bit, and every parameter gets an fp32 gradient."""
    dt = DTYPES[dt]
    torch.backends.cudnn.deterministic = True
    net = _block(pvb)
    x = torch.randn(2, 32, 19, 23, device=DEV).to(dt).requires_grad_()
    with torch.autocast("cuda", dtype=dt):
        y = net(x)
        d = net.conv(x)
        o1, o2, mk = torch.chunk(net.conv.conv_offset_mask(x), 3, dim=1)
    assert y.dtype == dt and d.dtype == dt
    c = net.conv
    explicit = pvb.dcn_v2_conv(x, torch.cat((o1, o2), 1), torch.sigmoid(mk), c.weight.to(dt), c.bias.to(dt), c.stride,
                               c.padding, c.dilation, c.deformable_groups)
    assert torch.equal(d, explicit)
    net.zero_grad()
    y.float().square().mean().backward()
    for name, p in net.named_parameters():
        assert p.grad is not None and p.grad.dtype == torch.float32, name
        assert bool(torch.isfinite(p.grad).all()) and float(p.grad.abs().sum()) > 0, name
    assert x.grad.dtype == dt


def test_fp16_grad_scaler_steps_and_skips_an_overflowing_step(pvb):
    """A GradScaler step goes through at an ordinary scale; at a scale that overflows fp16 the gradients hold inf, the
    scaler skips the step and lowers the scale."""
    net = _block(pvb)
    opt = torch.optim.SGD(net.parameters(), lr=1e-3)
    x = torch.randn(2, 32, 19, 23, device=DEV).half()

    def step(scaler):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            loss = net(x).float().square().mean()
        scaler.scale(loss).backward()
        before = [p.detach().clone() for p in net.parameters()]
        scaler.step(opt)
        scaler.update()
        return before

    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0)
    before = step(scaler)
    assert scaler.get_scale() == 1024.0
    assert any(not torch.equal(a, p) for a, p in zip(before, net.parameters()))
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 100)
    before = step(scaler)
    assert not all(bool(torch.isfinite(p.grad).all()) for p in net.parameters())
    assert scaler.get_scale() < 2.0 ** 100
    assert all(torch.equal(a, p) for a, p in zip(before, net.parameters()))


@pytest.mark.parametrize("dt", DT_IDS)
def test_deterministic_and_an_image_alone_equals_it_in_a_batch_of_16(pvb, dt):
    """Every detector layer at 512x512, a batch of 16: run to run bitwise equal, and images 0, 7 and 15 alone give
    their rows of the batch (the split-K factor depends on the image's shape only)."""
    dt = DTYPES[dt]
    for layer, c0 in enumerate(dc.DETECTOR["512x512"]):
        c = c0._replace(B=16)
        x, off, m, w, b = lowp(dc.make_inputs(c, seed=layer, offsets="random"), dt)
        o1, o2 = fwd(pvb, c, x, off, m, w, b), fwd(pvb, c, x, off, m, w, b)
        assert torch.equal(o1, o2), layer
        for i in (0, 7, 15):
            one = fwd(pvb, c._replace(B=1), x[i:i + 1], off[i:i + 1], m[i:i + 1], w, b)
            assert torch.equal(one, o1[i:i + 1]), (layer, i)


@pytest.mark.parametrize("dt", DT_IDS)
def test_no_host_sync_on_a_side_stream_and_forward_graph_capture(pvb, dt):
    dt = DTYPES[dt]
    case = dc.DETECTOR["544x736"][0]                      # a split-K layer
    x, off, m, w, b = lowp(dc.make_inputs(case, seed=6, offsets="random"), dt)
    wf, bf = w.float(), b.float()
    want = fwd(pvb, case, x, off, m, w, b)
    go = torch.randn_like(want)
    ts = [t.clone().requires_grad_() for t in (x, off, m, wf, bf)]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = pvb.dcn_v2_conv(*ts, case.stride, case.pad, case.dil, case.dg)
            grads = torch.autograd.grad(out, ts, go)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    s.synchronize()
    assert torch.equal(out, want) and all(bool(torch.isfinite(g).all()) for g in grads)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = fwd(pvb, case, x, off, m, w, b)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap, want)
