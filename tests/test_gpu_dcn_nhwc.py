"""GPU tests of the channels_last half-precision DCNv2 forward (pvb_dcn_forward_half_nhwc, csrc/dcn.cu; DESIGN.md
section 8o): its output is the NCHW call's bit for bit, channels_last, over the sweep and every detector shape, with
offset and mask in either layout; the backward of a channels_last call is the NCHW call's; a channels_last DeformConv
block runs under torch.autocast and a GradScaler; the call copies nothing but the weight; determinism, batch
independence, no host sync and graph capture."""
import pytest
import torch

import dcn_cases as dc
from test_gpu_dcn import DEV
from test_gpu_dcn_half import DT_IDS, DTYPES, _block, fwd, lowp

pytestmark = pytest.mark.gpu
CL = torch.channels_last
NCHW = torch.contiguous_format
LAYOUTS = {"cl": CL, "nchw": NCHW}

# the sweep has no case whose groups are a multiple of 8 channels wide, so these add the 16-byte sampler's: two groups
# of 8, and one group of 40 (a partial second chunk)
VEC = [dc.Case(2, 16, 7, 9, 5, 3, 3, (1, 1), (1, 1), (1, 1), 2),
       dc.Case(2, 40, 6, 11, 20, 3, 3, (2, 1), (1, 1), (1, 2), 1)]


def cl(t):
    return t.contiguous(memory_format=CL)


def assert_bitwise_channels_last(got, want):
    assert got.is_contiguous(memory_format=CL) and not got.is_contiguous()
    assert got.dtype == want.dtype and got.shape == want.shape
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
        float((got.float() - want.float()).abs().nan_to_num(0).max())


def check(pvb, c, x, off, m, w, b, op_layout):
    """x, off, m NCHW: the channels_last call (offset and mask in op_layout) against the NCHW call."""
    want = fwd(pvb, c, x, off, m, w, b)
    got = fwd(pvb, c, cl(x), *(t.contiguous(memory_format=op_layout) for t in (off, m)), w, b)
    assert_bitwise_channels_last(got, want)


SWEEP_CASES = [(c, "edges") for c in dc.SWEEP + VEC] + [(c, "random") for c in dc.SWEEP + VEC]


@pytest.mark.parametrize("lay", list(LAYOUTS))
@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case,offsets", SWEEP_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else v)
def test_sweep_equals_the_nchw_call_bit_for_bit(pvb, case, offsets, dt, lay):
    """Every edge of the bilinear domain, NaN / +-inf offsets on the small cases, both samplers (scalar and 16-byte)."""
    arrs = dc.make_inputs(case, seed=31, offsets=offsets, nonfinite=case.H * case.W < 1000)
    check(pvb, case, *lowp(arrs, DTYPES[dt]), LAYOUTS[lay])


def _random(c, B, dt, seed):
    """Detector-sized operands made on the device (the numpy generator is slow at a batch of 8)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    Ho, Wo = dc.out_hw(c)
    x = torch.randn((B, c.C, c.H, c.W), generator=g, device=DEV)
    off = torch.rand((B, 2 * c.dg * c.kh * c.kw, Ho, Wo), generator=g, device=DEV) * 5 - 2.5
    m = torch.rand((B, c.dg * c.kh * c.kw, Ho, Wo), generator=g, device=DEV)
    w = torch.randn((c.Co, c.C, c.kh, c.kw), generator=g, device=DEV) / (c.C * c.kh * c.kw) ** 0.5
    b = torch.randn((c.Co,), generator=g, device=DEV)
    return [t.to(dt) for t in (x, off, m, w, b)]


DETECTOR_CASES = [(key, layer) for key in dc.INPUTS for layer in range(len(dc.DETECTOR[key]))]


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("key,layer", DETECTOR_CASES, ids=lambda v: str(v))
def test_detector_layers_equal_the_nchw_call_bit_for_bit(pvb, key, layer, dt):
    """All 16 layers at the three input sizes, alone and in a batch of 8, offset and mask in both layouts."""
    c0 = dc.DETECTOR[key][layer]
    for B in (1, 8):
        c = c0._replace(B=B)
        ops = _random(c, B, DTYPES[dt], seed=layer)
        for lay in (CL, NCHW):
            check(pvb, c, *ops, lay)


@pytest.mark.parametrize("dt", DT_IDS)
def test_overflow_is_inf_and_an_empty_batch_is_channels_last(pvb, dt):
    dt = DTYPES[dt]
    case = VEC[1]
    x, off, m, w, b = lowp(dc.make_inputs(case, seed=4, offsets="zero"), dt)
    big = torch.finfo(dt).max
    for sign in (1, -1):
        check(pvb, case, torch.full_like(x, 1.0), off, torch.ones_like(m), torch.full_like(w, sign * big / 4),
              torch.zeros_like(b), CL)
        out = fwd(pvb, case, cl(torch.full_like(x, 1.0)), cl(off), cl(torch.ones_like(m)),
                  torch.full_like(w, sign * big / 4), torch.zeros_like(b))
        assert bool((out[:, :, 1:-1, 1:-1] == sign * float("inf")).all())
    e = case._replace(B=0)
    x0 = torch.empty((0, case.C, case.H, case.W), dtype=dt, device=DEV, memory_format=CL)
    y = fwd(pvb, e, x0, off[:0], m[:0], w, b)
    assert y.shape == (0, case.Co, *dc.out_hw(case)) and y.dtype == dt
    assert y.stride() == torch.empty(y.shape, memory_format=CL).stride()


GRAD_CASES = [dc.SWEEP[0], dc.SWEEP[2], dc.SWEEP[9]] + VEC


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case", GRAD_CASES, ids=dc.case_id)
def test_gradients_equal_the_nchw_call(pvb, monkeypatch, case, dt):
    """The same grad_output through dcn_v2_conv on channels_last and on NCHW operands of the same values: the backward
    gets bitwise equal operands, so grad_offset, grad_mask, grad_weight and grad_bias are bitwise equal; grad_input,
    summed with float atomics, is equal up to the order of those additions, as between two NCHW calls."""
    dt = DTYPES[dt]
    arrs = dc.make_inputs(case, seed=13, offsets="random")
    x, off, m = lowp(arrs[:3], dt)
    w, b = (torch.from_numpy(a).to(DEV) for a in arrs[3:])
    Ho, Wo = dc.out_hw(case)
    go = torch.randn((case.B, case.Co, Ho, Wo), device=DEV).to(dt)
    seen = []
    backward = pvb.dcn.dcn_backward
    monkeypatch.setattr(pvb.dcn, "dcn_backward", lambda *a, **k: seen.append(a) or backward(*a, **k))
    grads = []
    for layout in (NCHW, CL):
        ts = [t.detach().contiguous(memory_format=layout).requires_grad_() for t in (x, off, m)]
        ts += [t.clone().requires_grad_() for t in (w, b)]
        y = pvb.dcn_v2_conv(*ts, case.stride, case.pad, case.dil, case.dg)
        assert y.is_contiguous(memory_format=layout)
        grads.append(torch.autograd.grad(y, ts, go.contiguous(memory_format=layout)))
    for a0, a1 in zip(*seen):
        if isinstance(a0, torch.Tensor):
            assert torch.equal(a0.contiguous().view(torch.int32), a1.contiguous().view(torch.int32))
    names = ["grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"]
    for name, g0, g1 in zip(names, *grads):
        assert g0.dtype == g1.dtype, name
        if name == "grad_input":
            assert torch.allclose(g0.float(), g1.float(), rtol=1e-2, atol=1e-3), name
        else:
            assert torch.equal(g0, g1), name


@pytest.mark.parametrize("dt", DT_IDS)
def test_channels_last_deform_conv_block_under_autocast(pvb, dt):
    """A DeformConv block moved to channels_last, fed a channels_last input: the DCN's output is channels_last in the
    compute dtype and equals, bit for bit, an NCHW call on its own offset and mask; every parameter gets a finite fp32
    gradient."""
    dt = DTYPES[dt]
    torch.backends.cudnn.deterministic = True
    net = _block(pvb, chi=64, cho=64).to(memory_format=CL)
    xc = cl(torch.randn(2, 64, 19, 23, device=DEV).to(dt)).requires_grad_()
    with torch.autocast("cuda", dtype=dt):
        y = net(xc)
        d = net.conv(xc)
        o1, o2, mk = torch.chunk(net.conv.conv_offset_mask(xc), 3, dim=1)
    assert y.dtype == dt and y.is_contiguous(memory_format=CL)
    c = net.conv
    nchw = pvb.dcn_v2_conv(xc.detach().contiguous(), torch.cat((o1, o2), 1).contiguous(),
                           torch.sigmoid(mk).contiguous(), c.weight.to(dt), c.bias.to(dt), c.stride, c.padding,
                           c.dilation, c.deformable_groups)
    assert_bitwise_channels_last(d, nchw)
    net.zero_grad()
    y.float().square().mean().backward()
    for name, p in net.named_parameters():
        assert p.grad is not None and p.grad.dtype == torch.float32, name
        assert bool(torch.isfinite(p.grad).all()) and float(p.grad.abs().sum()) > 0, name
    assert xc.grad.dtype == dt


def test_fp16_grad_scaler_steps_and_skips_an_overflowing_step_channels_last(pvb):
    net = _block(pvb, chi=64, cho=64).to(memory_format=CL)
    opt = torch.optim.SGD(net.parameters(), lr=1e-3)
    x = cl(torch.randn(2, 64, 19, 23, device=DEV).half())

    def step(scaler):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            y = net(x)
            assert y.is_contiguous(memory_format=CL)
            loss = y.float().square().mean()
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
def test_a_channels_last_call_copies_nothing_but_the_weight(pvb, dt):
    """Operands already in the dtype and channels_last: two kernels, the weight's tap-major copy and the NHWC kernel."""
    c = dc.DETECTOR["512x512"][7]
    x, off, m, w, b = _random(c, 1, DTYPES[dt], seed=2)
    x, off, m = cl(x), cl(off), cl(m)
    fwd(pvb, c, x, off, m, w, b)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fwd(pvb, c, x, off, m, w, b)
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert len(kernels) == 2, kernels
    assert sum("dcn_forward_nhwc_kernel" in k for k in kernels) == 1, kernels


@pytest.mark.parametrize("dt", DT_IDS)
def test_deterministic_and_an_image_alone_equals_it_in_a_batch_of_16(pvb, dt):
    """Every detector layer at 512x512, a channels_last batch of 16: run to run bitwise equal, and images 0, 7 and 15
    alone give their rows of the batch."""
    for layer, c0 in enumerate(dc.DETECTOR["512x512"]):
        c = c0._replace(B=16)
        x, off, m, w, b = _random(c, 16, DTYPES[dt], seed=layer)
        x, off, m = cl(x), cl(off), cl(m)
        o1, o2 = fwd(pvb, c, x, off, m, w, b), fwd(pvb, c, x, off, m, w, b)
        assert o1.is_contiguous(memory_format=CL)
        assert torch.equal(o1.view(torch.int16), o2.view(torch.int16)), layer
        for i in (0, 7, 15):
            one = fwd(pvb, c._replace(B=1), x[i:i + 1], off[i:i + 1], m[i:i + 1], w, b)
            assert torch.equal(one.view(torch.int16), o1[i:i + 1].view(torch.int16)), (layer, i)


@pytest.mark.parametrize("dt", DT_IDS)
def test_no_host_sync_on_a_side_stream_and_forward_graph_capture(pvb, dt):
    dt = DTYPES[dt]
    case = dc.DETECTOR["544x736"][0]                      # a split-K layer
    x, off, m, w, b = _random(case, 1, dt, seed=6)
    x, off, m = cl(x), cl(off), cl(m)
    want = fwd(pvb, case, x, off, m, w, b)
    go = torch.randn_like(want)
    ts = [t.clone().requires_grad_() for t in (x, off, m, w.float(), b.float())]
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
    assert torch.equal(out, want) and out.is_contiguous(memory_format=CL)
    assert all(bool(torch.isfinite(g).all()) for g in grads)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = fwd(pvb, case, x, off, m, w, b)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap, want) and cap.is_contiguous(memory_format=CL)
