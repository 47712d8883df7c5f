"""GPU tests of DCNv2's TF32 path (pvb_dcn_forward_tf32 / pvb_dcn_backward_tf32, csrc/dcn.cu; DESIGN.md section 8p),
which dcn_v2_conv takes for fp32 inputs when torch allows TF32 matmuls: the forward's columns against the reference's
im2col (oracle/_ref/libdcn_ref.so) rounded once to TF32, bit for bit; the product and the five gradients within the
bounds DESIGN.md states; determinism; the fp16 / bf16 paths under the flag; and a DeformConv block under
set_float32_matmul_precision("high").  Every test that turns TF32 on restores torch's flags exactly."""
import numpy as np
import pytest
import torch
from torch import nn

import dcn_cases as dc
import dcn_oracle as do
from test_dcn_tf32_host import _restore_flags, _save_flags, tf32_rna
from test_gpu_dcn import DETECTOR_UNIQUE, DEV, U, gpu, ref_cols

pytestmark = pytest.mark.gpu
C_BOUND = 3          # DESIGN.md section 8p: |out - E| <= C_BOUND * K * u32 * (|b| + sum |W| |col|)
U_TF32 = 2.0 ** -11  # unit roundoff of the operands' rounding to TF32
HALF = {"f16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture
def tf32():
    """TF32 on through the new matmul flag for the test; the global and matmul flags restored exactly after it."""
    saved = _save_flags()
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    yield
    _restore_flags(saved)


def rna(t):
    """tf32_rna (cvt.rna.tf32.f32) of a CUDA fp32 tensor."""
    return torch.from_numpy(tf32_rna(t.cpu().numpy())).to(t.device)


def fwd(pvb, c, x, off, m, w, b):
    return pvb.dcn.dcn_forward(x, off, m, w, b, c.stride, c.pad, c.dil, c.dg)


def bwd(pvb, c, x, off, m, w, b, go, **kw):
    return pvb.dcn.dcn_backward(x, off, m, w, b, go, c.stride, c.pad, c.dil, c.dg, **kw)


IDENTITY_CASES = [(c, "edges") for c in dc.SWEEP] + [(c, "random") for c in dc.SWEEP] + \
                 [(c, "edges") for c in DETECTOR_UNIQUE]


@pytest.mark.parametrize("case,offsets", IDENTITY_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else v)
def test_identity_weight_returns_the_tf32_rounded_reference_columns_bit_for_bit(pvb, tf32, case, offsets):
    """W = I, bias 0: the output is tf32_rna of the reference im2col, exactly, at every edge of the bilinear domain,
    NaN / +-inf offsets (small sweep cases) and every detector shape at the three input sizes."""
    x, off, m, _, _ = dc.make_inputs(case, seed=21, offsets=offsets, nonfinite=case.H * case.W < 1000)
    wid, bid = dc.identity_weight(case)
    x, off, m, wid, bid = gpu(x, off, m, wid, bid)
    ours = fwd(pvb, case, x, off, m, wid, bid).reshape(case.B, wid.shape[0], -1)
    want = rna(ref_cols(case, x, off, m))
    torch.cuda.synchronize()
    assert torch.equal(ours, want), float((ours - want).abs().max())


def _patterns(n, rng):
    """fp32 bit patterns that pin the rounding: ties (both signs), values just around them, carries into the exponent,
    subnormals of every size, the smallest normals, zeros and ordinary values."""
    pats = [0x3F801000, 0xBF801000, 0x3F800FFF, 0x3F801001, 0x3FFFF000, 0xBFFFF000, 0x3F802000, 0x3F803000,
            0x00000001, 0x00000FFF, 0x00001000, 0x80001000, 0x00002FFF, 0x007FF000, 0x007FFFFF, 0x80400000,
            0x00800000, 0x80800000, 0x00801000, 0x00000000, 0x80000000]
    u = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    u = np.where((u & 0x7F800000) == 0x7F800000, u & 0x807FFFFF, u)          # no inf / NaN
    u[:len(pats)] = pats
    sub = rng.integers(1, 1 << 23, n // 4, dtype=np.uint64).astype(np.uint32)
    u[len(pats):len(pats) + len(sub)] = sub | (rng.integers(0, 2, len(sub), dtype=np.uint64).astype(np.uint32) << 31)
    return u.view(np.float32)


def toward_zero(v):
    """fp64 values rounded to fp32 toward zero, except that a value beyond the fp32 range is +-inf, as the tensor
    cores return it."""
    v = v.cpu().numpy()
    with np.errstate(over="ignore"):
        f = v.astype(np.float32)
    over = np.isfinite(f) & (np.abs(f.astype(np.float64)) > np.abs(v))
    f[over] = np.nextafter(f[over], np.float32(0))
    return torch.from_numpy(f).to(DEV)


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 20, 2.0 ** -20], ids=["one", "2^20", "2^-20"])
def test_zero_offsets_pin_the_device_rounding_on_chosen_bit_patterns(pvb, tf32, scale):
    """Zero offsets and mask 1: the columns are the input itself.  With W = scale * I the output is
    RZ_fp32(scale * tf32_rna(x)): subnormal operands (scale 1, 2^20) are kept, not flushed, and so are subnormal
    products (2^-20), which the tensor cores round toward zero (a product too small for the smallest subnormal gives
    0).  A product beyond the fp32 range (2^20) is +-inf.  Every other product is exact, so the output is
    scale * tf32_rna(x) itself."""
    case = dc.Case(2, 8, 11, 13, 72, 3, 3, (1, 1), (1, 1), (1, 1), 1)
    rng = np.random.default_rng(7)
    x = _patterns(case.B * case.C * case.H * case.W, rng).reshape(case.B, case.C, case.H, case.W)
    Ho, Wo = dc.out_hw(case)
    off = np.zeros((case.B, 18, Ho, Wo), np.float32)
    m = np.ones((case.B, 9, Ho, Wo), np.float32)
    wid, bid = dc.identity_weight(case)
    x, off, m, wid, bid = gpu(x, off, m, wid * np.float32(scale), bid)
    ours = fwd(pvb, case, x, off, m, wid, bid).reshape(case.B, wid.shape[0], -1)
    cols = ref_cols(case, x, off, m)
    want = toward_zero(rna(cols).double() * scale)
    torch.cuda.synchronize()
    bad = ours.view(torch.int32) != want.view(torch.int32)
    zero_eq = (ours == 0) & (want == 0)                     # +0 from the sum where the column is -0
    bad &= ~zero_eq
    assert not bool(bad.any()), (int(bad.sum()), ours[bad][:8].tolist(), want[bad][:8].tolist(), cols[bad][:8].tolist())


FWD_CASES = [(c, 1) for c in dc.SWEEP] + [(c._replace(B=8), 8) for c in dc.SWEEP[:4]] + \
            [(c, 1) for c in DETECTOR_UNIQUE if c.H * c.W <= 92 * 68] + [(dc.DETECTOR["512x512"][0]._replace(B=8), 8)]


@pytest.mark.parametrize("case,B", FWD_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else f"B{v}")
def test_forward_with_real_weights_is_within_the_tf32_bound(pvb, tf32, case, B):
    """E = fp64(b + RN(W) RN(col)) on the TF32-rounded operands: ours within C_BOUND * K * u32 * (|b| + |RN W| |RN col|).
    Against fp64(b + W col) on the unrounded operands, the operand rounding (2 u_tf32 + u_tf32^2) |W| |col| is added;
    torch.matmul under TF32 on the reference's columns meets that bound too."""
    x, off, m, w, b = gpu(*dc.make_inputs(case, seed=3, offsets="random"))
    ours = fwd(pvb, case, x, off, m, w, b).reshape(case.B, case.Co, -1).double()
    cols = ref_cols(case, x, off, m)
    W2 = w.reshape(case.Co, -1)
    K = case.C * case.kh * case.kw
    Wr, cr = rna(W2).double(), rna(cols).double()
    exact_r = b.double()[None, :, None] + torch.matmul(Wr, cr)
    abs_r = b.double().abs()[None, :, None] + torch.matmul(Wr.abs(), cr.abs())
    assert bool(((ours - exact_r).abs() <= C_BOUND * K * U * abs_r).all()), \
        float(((ours - exact_r).abs() / abs_r.clamp_min(1e-300)).max() / (C_BOUND * K * U))
    exact = b.double()[None, :, None] + torch.matmul(W2.double(), cols.double())
    prod_abs = torch.matmul(W2.double().abs(), cols.double().abs())
    loose = C_BOUND * K * U * abs_r + (2 * U_TF32 + U_TF32 ** 2) * prod_abs
    theirs = (b[None, :, None] + torch.matmul(W2, cols)).double()             # cuBLAS, TF32 on
    assert bool(((ours - exact).abs() <= loose).all())
    assert bool(((theirs - exact).abs() <= loose).all()), float(((theirs - exact).abs() / loose.clamp_min(1e-300)).max())


BWD_CASES = [(c, "random") for c in dc.SWEEP] + [(c, "edges") for c in dc.SWEEP[:5]]


@pytest.mark.parametrize("case,offsets", BWD_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else v)
def test_backward_is_within_the_tf32_bounds_of_the_restatement(pvb, tf32, case, offsets):
    """The five gradients against the fp64 restatement on RN(W) and RN(grad_out), the operands the TF32 grad_cols
    multiplies: grad_cols adds each term with up to 2 u32 of error, so its chain counts twice in grad_input / offset /
    mask; grad_weight adds the TF32 rounding of its re-sampled columns, u_tf32 of its terms.  grad_bias is the IEEE
    path's bit for bit; nothing but grad_input depends on the chunking of grad_cols."""
    arrs = dc.make_inputs(case, seed=9, offsets=offsets)
    Ho, Wo = dc.out_hw(case)
    go = np.random.default_rng(4).standard_normal((case.B, case.Co, Ho, Wo)).astype(np.float32)
    x, off, m, w, b = arrs
    want = do.backward(x, off, m, tf32_rna(w), b, tf32_rna(go), case.stride, case.pad, case.dil, case.dg)
    t = gpu(*arrs, go)
    got = bwd(pvb, case, *t)
    got1 = bwd(pvb, case, *t, max_column_bytes=1)
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    ieee = bwd(pvb, case, *t)
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    assert torch.equal(got[4], ieee[4])
    Cg = case.C // case.dg
    chains = dict(grad_input=2 * case.Co + 8 + want["grad_input_terms"], grad_offset=2 * case.Co + Cg + 16,
                  grad_mask=2 * case.Co + Cg + 8, grad_weight=C_BOUND * (case.B * Ho * Wo + 8))
    for i, name in enumerate(["grad_input", "grad_offset", "grad_mask", "grad_weight"]):
        g = got[i].double().cpu().numpy()
        if name != "grad_input":
            assert torch.equal(got[i], got1[i]), name
        rel = chains[name] * U + (U_TF32 * (1 + 16 * U) if name == "grad_weight" else 0.0)
        bound = rel * want[name + "_abs"] * 1.01 + 1e-30
        err = np.abs(g - want[name])
        assert (err <= bound).all(), (name, float((err / bound).max()))


def test_deterministic_and_an_image_alone_equals_it_in_a_batch_of_16(pvb, tf32):
    """Every detector layer at 512x512: the forward of a batch of 16 is run-to-run bitwise equal and images 0, 7 and 15
    alone give their rows; the backward (B = 2) is run-to-run equal and does not depend on max_column_bytes."""
    for layer, c0 in enumerate(dc.DETECTOR["512x512"]):
        c = c0._replace(B=16)
        x, off, m, w, b = gpu(*dc.make_inputs(c, seed=layer, offsets="random"))
        o1, o2 = fwd(pvb, c, x, off, m, w, b), fwd(pvb, c, x, off, m, w, b)
        assert torch.equal(o1, o2), layer
        for i in (0, 7, 15):
            one = c._replace(B=1)
            assert torch.equal(fwd(pvb, one, x[i:i + 1], off[i:i + 1], m[i:i + 1], w, b), o1[i:i + 1]), (layer, i)
        c2 = c._replace(B=2)
        t = (x[:2], off[:2], m[:2], w, b, torch.randn_like(o1[:2]))
        g1, g2, g3 = bwd(pvb, c2, *t), bwd(pvb, c2, *t), bwd(pvb, c2, *t, max_column_bytes=1)
        for k in range(1, 5):
            assert torch.equal(g1[k], g2[k]) and torch.equal(g1[k], g3[k]), (layer, k)


@pytest.mark.parametrize("dt", list(HALF))
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_half_forward_ignores_the_flag_and_its_backward_follows_it(pvb, dt, layout):
    """fp16 / bf16: the forward with TF32 on is bitwise the forward with it off; the backward with it on is
    dcn_backward (the TF32 entry) on the up-cast operands, bit for bit but grad_input."""
    dt = HALF[dt]
    case = dc.SWEEP[8]._replace(B=2)
    arrs = dc.make_inputs(case, seed=9, offsets="random")
    lay = torch.channels_last if layout == "channels_last" else torch.contiguous_format
    x, off, m = (t.to(dt).contiguous(memory_format=lay) for t in gpu(*arrs[:3]))
    w, b = gpu(*arrs[3:])
    st = (case.stride, case.pad, case.dil, case.dg)
    ieee_out = pvb.dcn_v2_conv(x, off, m, w, b, *st)
    saved = _save_flags()
    try:
        torch.backends.cuda.matmul.fp32_precision = "tf32"
        ts = [t.clone().requires_grad_() for t in (x, off, m, w, b)]
        y = pvb.dcn_v2_conv(*ts, *st)
        assert torch.equal(y.view(torch.int16), ieee_out.view(torch.int16))
        go = torch.randn_like(y)
        got = torch.autograd.grad(y, ts, go)
        up = [t.float() for t in (x, off, m, w.to(dt), b.to(dt), go)]
        want = pvb.dcn.dcn_backward(*up, *st)
        for k in range(1, 5):
            assert torch.equal(got[k], want[k].to(ts[k].dtype)), k
    finally:
        _restore_flags(saved)
    ieee = pvb.dcn.dcn_backward(*up, *st)
    assert torch.equal(ieee[4], want[4]) and not torch.equal(ieee[3], want[3])


class DeformConvBlock(nn.Module):
    """The shape of lib/networks/ct/dla_dcn.py's DeformConv: DCN 3x3 -> BatchNorm -> ReLU."""

    def __init__(self, pvb, chi, cho):
        super().__init__()
        self.conv = pvb.DCN(chi, cho, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)
        self.actf = nn.Sequential(nn.BatchNorm2d(cho), nn.ReLU(inplace=True))

    def forward(self, x):
        return self.actf(self.conv(x))


def _kernels(pvb, net, x):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        net(x).square().mean().backward()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_deform_conv_block_under_high_matmul_precision(pvb, layout):
    """An fp32 DeformConv block under set_float32_matmul_precision("high"): every parameter gets a finite gradient, one
    SGD step changes them, and the TF32 kernels run with the flag on, the FFMA ones with it off."""
    torch.manual_seed(0)
    net = DeformConvBlock(pvb, 32, 24).to(DEV)
    with torch.no_grad():
        net.conv.conv_offset_mask.weight.normal_(0, 0.05)
        net.conv.conv_offset_mask.bias.normal_(0, 0.5)
        net.conv.bias.normal_()
    lay = torch.channels_last if layout == "channels_last" else torch.contiguous_format
    net = net.to(memory_format=lay)
    x = torch.randn(2, 32, 19, 23, device=DEV).contiguous(memory_format=lay).requires_grad_()
    tf32_names = ("dcn_forward_tf32_kernel", "dcn_grad_cols_tf32_kernel", "dcn_grad_weight_tf32_kernel")
    ffma_names = ("dcn_forward_kernel", "dcn_grad_cols_kernel", "dcn_grad_weight_kernel")
    saved = _save_flags()
    try:
        torch.set_float32_matmul_precision("high")
        before = [p.detach().clone() for p in net.parameters()]
        opt = torch.optim.SGD(net.parameters(), lr=0.1)
        opt.zero_grad()
        kernels = _kernels(pvb, net, x)
        for name, p in net.named_parameters():
            assert p.grad is not None and bool(torch.isfinite(p.grad).all()), name
        opt.step()
        for (name, p), p0 in zip(net.named_parameters(), before):
            if name != "conv.bias":            # BatchNorm cancels a per-channel shift: its gradient is 0 up to rounding
                assert not torch.equal(p0, p), name
        for k in tf32_names:
            assert sum(k in e for e in kernels) == 1, (k, kernels)
        assert not any(k in e for e in kernels for k in ffma_names), kernels
    finally:
        _restore_flags(saved)
    kernels = _kernels(pvb, net, x)
    assert not any("dcn_" in e and "tf32" in e for e in kernels), kernels
    for k in ffma_names:
        assert sum(k in e for e in kernels) == 1, (k, kernels)


def test_no_host_sync_on_a_side_stream_and_forward_graph_capture(pvb, tf32):
    case = dc.SWEEP[1]
    x, off, m, w, b = gpu(*dc.make_inputs(case, seed=6, offsets="random"))
    want = fwd(pvb, case, x, off, m, w, b)
    go = torch.randn_like(want)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = fwd(pvb, case, x, off, m, w, b)
            grads = bwd(pvb, case, x, off, m, w, b, go)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    s.synchronize()
    assert torch.equal(out, want) and all(torch.isfinite(g).all() for g in grads)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = fwd(pvb, case, x, off, m, w, b)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap, want)
