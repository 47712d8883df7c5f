"""GPU tests of the DCNv2 kernels (csrc/dcn.cu) against the reference's own sampling kernels (oracle/_ref/libdcn_ref.so,
the unmodified dcn_v2_im2col_cuda.cu) and the fp64 restatement (oracle/dcn_oracle.py), at the sweep of
tests/dcn_cases.py and every DLA-34 detector shape."""
import ctypes
import os

import numpy as np
import pytest
import torch

import dcn_cases as dc
import dcn_oracle as do

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libdcn_ref.so")
U = 2.0 ** -24
DEV = "cuda:0"


def gamma(n):
    return n * U / (1 - n * U)


_REF = None


def ref():
    global _REF
    if _REF is None:
        if not os.path.exists(REF_LIB):
            pytest.skip("oracle/_ref/libdcn_ref.so not built (no clean-pvnet checkout at build time)")
        lib = ctypes.CDLL(REF_LIB)
        i, p = ctypes.c_int, ctypes.c_void_p
        lib.modulated_deformable_im2col_cuda.argtypes = [p, p, p, p] + [i] * 15 + [p]
        lib.modulated_deformable_col2im_cuda.argtypes = [p, p, p, p] + [i] * 15 + [p]
        lib.modulated_deformable_col2im_coord_cuda.argtypes = [p, p, p, p, p] + [i] * 15 + [p, p]
        for f in ("modulated_deformable_im2col_cuda", "modulated_deformable_col2im_cuda",
                  "modulated_deformable_col2im_coord_cuda"):
            getattr(lib, f).restype = None
        _REF = lib
    return _REF


def _geom(c):
    Ho, Wo = dc.out_hw(c)
    return [c.C, c.H, c.W, Ho, Wo, c.kh, c.kw, c.pad[0], c.pad[1], c.stride[0], c.stride[1], c.dil[0], c.dil[1], c.dg]


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ref_cols(c, x, off, m):
    """The reference im2col, one image at a time as its backward runs it: [B, C*kh*kw, Ho*Wo]."""
    Ho, Wo = dc.out_hw(c)
    out = torch.empty((c.B, c.C * c.kh * c.kw, Ho * Wo), device=DEV)
    for b in range(c.B):
        ref().modulated_deformable_im2col_cuda(_stream(), _ptr(x[b]), _ptr(off[b]), _ptr(m[b]), 1, *_geom(c), _ptr(out[b]))
    return out


def gpu(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in arrays]


def run_forward(pvb, c, x, off, m, w, b):
    return pvb.dcn.dcn_forward(x, off, m, w, b, c.stride, c.pad, c.dil, c.dg)


def run_backward(pvb, c, x, off, m, w, b, go, **kw):
    return pvb.dcn.dcn_backward(x, off, m, w, b, go, c.stride, c.pad, c.dil, c.dg, **kw)


DETECTOR_UNIQUE = sorted({c for cases in dc.DETECTOR.values() for c in cases})
IDENTITY_CASES = [(c, "edges") for c in dc.SWEEP] + [(c, "random") for c in dc.SWEEP] + \
                 [(c, "edges") for c in DETECTOR_UNIQUE]


@pytest.mark.parametrize("case,offsets", IDENTITY_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else v)
def test_identity_weight_returns_the_reference_columns_bit_for_bit(pvb, case, offsets):
    """With W = I (C_out = C*kh*kw) and bias 0 the fused forward returns the columns; they equal the reference im2col
    kernel's exactly, at sample points on every edge of the bilinear domain (and NaN / +-inf offsets in the sweep)."""
    x, off, m, _, _ = dc.make_inputs(case, seed=21, offsets=offsets, nonfinite=case.H * case.W < 1000)
    wid, bid = dc.identity_weight(case)
    x, off, m, wid, bid = gpu(x, off, m, wid, bid)
    ours = run_forward(pvb, case, x, off, m, wid, bid).reshape(case.B, wid.shape[0], -1)
    want = ref_cols(case, x, off, m)
    torch.cuda.synchronize()
    assert torch.equal(ours, want), float((ours - want).abs().max())


FWD_CASES = [(c, 1) for c in dc.SWEEP] + [(c._replace(B=8), 8) for c in dc.SWEEP[:4]] + \
            [(c, 1) for c in DETECTOR_UNIQUE if c.H * c.W <= 92 * 68] + [(dc.DETECTOR["512x512"][0]._replace(B=8), 8)]


@pytest.mark.parametrize("case,B", FWD_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else f"B{v}")
def test_forward_with_real_weights_is_within_the_fp32_dot_product_bound(pvb, case, B):
    """|ours - fp64(b + W cols_ref)| <= gamma_{K+1} (|b| + |W| |cols_ref|), K = C*kh*kw; the reference's own algorithm
    (its columns + fp32 matmul, TF32 off) meets the same bound, so it is a fair one."""
    x, off, m, w, b = gpu(*dc.make_inputs(case, seed=3, offsets="random"))
    ours = run_forward(pvb, case, x, off, m, w, b).reshape(case.B, case.Co, -1).double()
    cols = ref_cols(case, x, off, m)
    W2 = w.reshape(case.Co, -1)
    exact = b.double()[None, :, None] + torch.matmul(W2.double(), cols.double())
    absb = b.double().abs()[None, :, None] + torch.matmul(W2.double().abs(), cols.double().abs())
    K = case.C * case.kh * case.kw
    bound = gamma(K + 1) * absb
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        theirs = (b[None, :, None] + torch.matmul(W2, cols)).double()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert bool(((ours - exact).abs() <= bound).all()), float(((ours - exact).abs() / bound.clamp_min(1e-300)).max())
    assert bool(((theirs - exact).abs() <= bound).all())


BWD_CASES = [(c, "random") for c in dc.SWEEP] + [(c, "edges") for c in dc.SWEEP]


def _chains(c):
    Ho, Wo = dc.out_hw(c)
    Cg = c.C // c.dg
    return dict(grad_cols=c.Co, grad_mask=c.Co + Cg + 8, grad_offset=c.Co + Cg + 16, grad_weight=c.B * Ho * Wo + 8,
                grad_bias=c.B * Ho * Wo)


@pytest.mark.parametrize("case,offsets", BWD_CASES, ids=lambda v: dc.case_id(v) if isinstance(v, tuple) else v)
def test_backward_is_within_the_rounding_bound_of_the_restatement(pvb, case, offsets):
    """All five gradients against the fp64 restatement, within n*u*(sum of |terms|), n the longest accumulation
    chain of each; the result does not depend on the image chunking of grad_cols."""
    arrs = dc.make_inputs(case, seed=9, offsets=offsets)
    Ho, Wo = dc.out_hw(case)
    go = np.random.default_rng(4).standard_normal((case.B, case.Co, Ho, Wo)).astype(np.float32)
    want = do.backward(*arrs, go, case.stride, case.pad, case.dil, case.dg)
    t = gpu(*arrs, go)
    got = run_backward(pvb, case, *t)
    got1 = run_backward(pvb, case, *t, max_column_bytes=1)        # one image per chunk
    names = ["grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"]
    chains = _chains(case)
    for name, g, g1 in zip(names, got, got1):
        g = g.double().cpu().numpy()
        if name == "grad_input":
            n = case.Co + 8 + want["grad_input_terms"]
        else:
            n = chains[name]
            assert np.array_equal(g, g1.double().cpu().numpy()), name
        err = np.abs(g - want[name])
        bound = n * U * want[name + "_abs"] * 1.01 + 1e-30
        assert (err <= bound).all(), (name, float((err / bound).max()))


@pytest.mark.parametrize("case", [c for c in dc.SWEEP if c.pad[0] == c.pad[1]] + DETECTOR_UNIQUE[:3], ids=dc.case_id)
def test_backward_identity_weight_matches_the_reference_col2im_kernels(pvb, case):
    """With W = I the backward's grad_cols is grad_out exactly, so grad_offset / grad_mask / grad_input can be set
    against the reference's col2im_coord / col2im launchers run on grad_out; both sides meet the restatement's bound.
    (The reference's col2im launcher passes pad_h for pad_w, so only square padding is compared.)"""
    x, off, m, _, _ = dc.make_inputs(case, seed=5, offsets="random")
    wid, bid = dc.identity_weight(case)
    K = wid.shape[0]
    Ho, Wo = dc.out_hw(case)
    go = np.random.default_rng(8).standard_normal((case.B, K, Ho, Wo)).astype(np.float32)
    tx, toff, tm, tw, tb, tgo = gpu(x, off, m, wid, bid, go)
    gi, goff, gm, _, _ = run_backward(pvb, case, tx, toff, tm, tw, tb, tgo)
    rgi, rgoff, rgm = torch.zeros_like(tx), torch.zeros_like(toff), torch.zeros_like(tm)
    for b in range(case.B):
        ref().modulated_deformable_col2im_coord_cuda(_stream(), _ptr(tgo[b]), _ptr(tx[b]), _ptr(toff[b]), _ptr(tm[b]), 1,
                                                     *_geom(case), _ptr(rgoff[b]), _ptr(rgm[b]))
        ref().modulated_deformable_col2im_cuda(_stream(), _ptr(tgo[b]), _ptr(toff[b]), _ptr(tm[b]), 1, *_geom(case),
                                               _ptr(rgi[b]))
    torch.cuda.synchronize()
    if case.H * case.W * case.C > 200000:
        pairs = [("grad_offset", goff, rgoff), ("grad_mask", gm, rgm), ("grad_input", gi, rgi)]
        for name, a, r in pairs:       # too large for the restatement: ours against the reference, relative
            scale = float(r.abs().max()) + 1e-30
            assert float((a - r).abs().max()) <= 1e-5 * scale, name
        return
    want = do.backward(x, off, m, wid, bid, go, case.stride, case.pad, case.dil, case.dg)
    Cg = case.C // case.dg
    for name, a, r in [("grad_offset", goff, rgoff), ("grad_mask", gm, rgm), ("grad_input", gi, rgi)]:
        n = (8 + want["grad_input_terms"]) if name == "grad_input" else Cg + 16
        bound = n * U * want[name + "_abs"] * 1.01 + 1e-30
        for side in (a, r):
            err = np.abs(side.double().cpu().numpy() - want[name])
            assert (err <= bound).all(), (name, float((err / bound).max()))


def test_forward_and_backward_are_deterministic_and_images_independent(pvb):
    case = dc.SWEEP[8]._replace(B=4)
    x, off, m, w, b = gpu(*dc.make_inputs(case, seed=1, offsets="random"))
    o1, o2 = run_forward(pvb, case, x, off, m, w, b), run_forward(pvb, case, x, off, m, w, b)
    assert torch.equal(o1, o2)
    for i in range(case.B):
        one = case._replace(B=1)
        alone = run_forward(pvb, one, x[i:i + 1], off[i:i + 1], m[i:i + 1], w, b)
        assert torch.equal(alone, o1[i:i + 1])
    go = torch.randn_like(o1)
    g1 = run_backward(pvb, case, x, off, m, w, b, go)
    g2 = run_backward(pvb, case, x, off, m, w, b, go)
    for a, c in zip(g1[1:], g2[1:]):
        assert torch.equal(a, c)
    big = dc.DETECTOR["512x512"][7]._replace(B=2)
    x, off, m, w, b = gpu(*dc.make_inputs(big, seed=2, offsets="random"))
    go = torch.randn((2, big.Co, big.H, big.W), device=DEV)
    g1 = run_backward(pvb, big, x, off, m, w, b, go)
    g2 = run_backward(pvb, big, x, off, m, w, b, go)
    for a, c in zip(g1[1:], g2[1:]):
        assert torch.equal(a, c)


def test_no_host_sync_on_a_side_stream_and_forward_graph_capture(pvb):
    case = dc.SWEEP[1]
    x, off, m, w, b = gpu(*dc.make_inputs(case, seed=6, offsets="random"))
    want = run_forward(pvb, case, x, off, m, w, b)
    go = torch.randn_like(want)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = run_forward(pvb, case, x, off, m, w, b)
            grads = run_backward(pvb, case, x, off, m, w, b, go)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    s.synchronize()
    assert torch.equal(out, want) and all(torch.isfinite(g).all() for g in grads)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = run_forward(pvb, case, x, off, m, w, b)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap, want)


def test_dcn_module_matches_the_functional_form_and_fills_every_gradient(pvb):
    torch.manual_seed(0)
    net = pvb.DCN(24, 16, kernel_size=(3, 3), stride=1, padding=1, deformable_groups=2).to(DEV)
    with torch.no_grad():
        net.conv_offset_mask.weight.normal_(0, 0.05)
        net.conv_offset_mask.bias.normal_(0, 0.5)
        net.bias.normal_()
    x = torch.randn(2, 24, 11, 13, device=DEV, requires_grad=True)
    y = net(x)
    out = net.conv_offset_mask(x)
    o1, o2, mk = torch.chunk(out, 3, dim=1)
    y2 = pvb.dcn_v2_conv(x, torch.cat((o1, o2), 1), torch.sigmoid(mk), net.weight, net.bias, net.stride, net.padding,
                         net.dilation, net.deformable_groups)
    assert torch.equal(y, y2)
    go = torch.randn_like(y)
    params = [net.weight, net.bias, net.conv_offset_mask.weight, net.conv_offset_mask.bias]
    grads = torch.autograd.grad(y, [x] + params, go, retain_graph=True)
    grads2 = torch.autograd.grad(y2, [x] + params, go)
    assert torch.equal(grads[1], grads2[1]) and torch.equal(grads[2], grads2[2])
    for a, b in zip(grads[:1] + grads[3:], grads2[:1] + grads2[3:]):     # through grad_input / cuDNN's conv backward
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5)
    net.zero_grad()
    (y * go).sum().backward()
    for name, p in net.named_parameters():
        assert p.grad is not None and float(p.grad.abs().sum()) > 0, name
    # a non-contiguous input is made contiguous, not misread
    xt = x.detach().transpose(2, 3).contiguous().transpose(2, 3)
    assert not xt.is_contiguous()
    assert torch.equal(net(xt), net(x.detach()))
