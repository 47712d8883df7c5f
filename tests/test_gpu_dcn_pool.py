"""GPU tests of the deformable PSROI pooling kernels (csrc/dcn_pool.cu) against the reference's own kernels
(oracle/_ref/libdcn_pool_ref.so, the unmodified dcn_v2_psroi_pooling_cuda.cu) and the fp64 restatement
(oracle/dcn_pool_oracle.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import dcn_pool_oracle as po

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libdcn_pool_ref.so")
U = 2.0 ** -24
DEV = "cuda:0"
_REF = None


def ref():
    global _REF
    if _REF is None:
        if not os.path.exists(REF_LIB):
            pytest.skip("oracle/_ref/libdcn_pool_ref.so not built (no clean-pvnet checkout at build time)")
        lib = ctypes.CDLL(REF_LIB)
        i, p, f = ctypes.c_int, ctypes.c_void_p, ctypes.c_float
        lib.ref_dcn_pool_forward.argtypes = [p] * 5 + [i] * 9 + [f, f, p]
        lib.ref_dcn_pool_backward.argtypes = [p] * 7 + [i] * 9 + [f, f, p]
        lib.ref_dcn_pool_forward.restype = lib.ref_dcn_pool_backward.restype = None
        _REF = lib
    return _REF


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def make(seed, B=2, C=32, H=64, W=64, n=20, P=7, ps=None, spp=4, nc=1, scale=0.25, std=0.1, span=256, size=64,
         trans_scale=1.0):
    """test.py's example_dpooling inputs, generalised: batch in [0, B), corners random integers."""
    g = torch.Generator().manual_seed(seed)
    ps = P if ps is None else ps
    x = torch.randn(B, C, H, W, generator=g)
    b = torch.randint(B, (n, 1), generator=g).float()
    xy = torch.randint(span, (n, 2), generator=g).float()
    wh = torch.randint(size, (n, 2), generator=g).float()
    rois = torch.cat((b, xy, xy + wh), 1)
    trans = torch.randn(n, 2 * nc, ps, ps, generator=g) * trans_scale
    return dict(x=x.to(DEV), rois=rois.to(DEV), trans=trans.to(DEV),
                kw=dict(spatial_scale=scale, pooled_size=P, output_dim=C, group_size=1, part_size=ps,
                        sample_per_part=spp, trans_std=std))


def ours_fwd(c, no_trans):
    return pvb_mod().dcn_pool.pool_forward(c["x"], c["rois"], c["trans"], no_trans=no_trans, **c["kw"])


def ours_bwd(c, go, no_trans):
    return pvb_mod().dcn_pool.pool_backward(go, c["x"], c["rois"], c["trans"], no_trans=no_trans, **c["kw"])


def _geom(c, no_trans):
    k = c["kw"]
    B, C, H, W = c["x"].shape
    nc = 1 if no_trans else c["trans"].shape[1] // 2
    return [c["rois"].shape[0], C, H, W, k["pooled_size"], k["part_size"], k["sample_per_part"], nc, int(no_trans),
            ctypes.c_float(k["spatial_scale"]), ctypes.c_float(k["trans_std"])]


def ref_fwd(c, no_trans):
    n, C, P = c["rois"].shape[0], c["x"].shape[1], c["kw"]["pooled_size"]
    out = torch.zeros((n, C, P, P), device=DEV)
    cnt = torch.zeros_like(out)
    g = _geom(c, no_trans)
    ref().ref_dcn_pool_forward(_p(c["x"]), _p(c["rois"]), _p(c["trans"]), _p(out), _p(cnt), *g, _s())
    return out, cnt


def ref_bwd(c, go, cnt, no_trans):
    gi, gt = torch.zeros_like(c["x"]), torch.zeros_like(c["trans"])
    g = _geom(c, no_trans)
    ref().ref_dcn_pool_backward(_p(go), _p(cnt), _p(c["x"]), _p(c["rois"]), _p(c["trans"]), _p(gi), _p(gt), *g, _s())
    return gi, gt


_PVB = None


def pvb_mod():
    global _PVB
    if _PVB is None:
        import clean_pvnet_b200
        _PVB = clean_pvnet_b200
    return _PVB


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _edit(c, rois=None, trans=None):
    c = dict(c)
    if rois is not None:
        c["rois"] = torch.tensor(rois, dtype=torch.float32, device=DEV)
    if trans is not None:
        c["trans"] = trans
    return c


def sweep():
    cases = {}
    cases["example_dpooling"] = make(1)
    cases["example_mdpooling"] = make(2)
    cases["gradient_dpooling"] = make(3, B=2, C=3, H=5, W=5, n=4, P=3, span=15, size=10, std=0.0)
    zero = make(4, B=2, C=16, H=64, W=64, n=2, std=0.0)
    zero["x"].zero_()
    zero["x"][0, :, 16:26, 16:26] = 1
    zero["x"][1, :, 10:20, 20:30] = 2
    cases["pooling_zero_offset"] = _edit(zero, rois=[[0, 65, 65, 103, 103], [1, 81, 41, 119, 79]],
                                         trans=torch.zeros(2, 2, 7, 7, device=DEV))
    for spp in (2, 4):
        cases[f"detector_head_spp{spp}"] = make(5 + spp, B=2, C=256, H=50, W=68, n=1024, scale=1 / 16, spp=spp,
                                                span=900, size=400)
    cases["part_size_5"] = make(10, ps=5)
    cases["part_size_9"] = make(11, ps=9)
    cases["classes_2"] = make(12, nc=2)
    cases["classes_4"] = make(13, nc=4, ps=4)
    cases["spp_1"] = make(14, spp=1)
    cases["spp_8"] = make(15, spp=8)
    cases["spp_32"] = make(16, spp=32, n=3, C=8)
    cases["scale_1"] = make(17, scale=1.0, span=60, size=30)
    cases["scale_1_32"] = make(18, scale=1 / 32, span=2000, size=1500)
    cases["P_11_big_bins"] = make(19, P=11, ps=3, spp=6)
    base = make(20, n=8)
    cases["outside"] = _edit(base, rois=[[0, 300, 300, 400, 400], [1, -200, -200, -100, -100], [0, 1000, 0, 1100, 50],
                                         [1, 0, -90, 50, -20], [0, -5, 10, -3, 12], [1, 258, 258, 260, 260],
                                         [0, 0, 300, 40, 320], [1, 300, 0, 320, 40]])
    cases["borders"] = _edit(base, rois=[[0, 0, 0, 255, 255], [1, 0, 0, 3, 255], [0, 252, 0, 255, 255],
                                         [1, 0, 252, 255, 255], [0, 0, 0, 255, 3], [1, -2, -2, 2, 2],
                                         [0, 253, 253, 258, 258], [1, 0, 0, 0, 0]])
    cases["degenerate"] = _edit(base, rois=[[0, 50, 50, 40, 40], [1, 10, 10, 10, 10], [0, 60, 20, 59, 80],
                                            [1, 30, 90, 90, 30], [0, 10.4, 10.4, 10.4, 10.4], [1, 5, 5, 4.6, 4.6],
                                            [0, 100, 100, 0, 0], [1, 200, 200, 199.5, 199.5]])
    cases["half_corners"] = _edit(base, rois=[[0, 10.5, 20.5, 60.5, 80.5], [1, -0.5, -1.5, 2.5, 3.5],
                                              [0, 0.5, 0.5, 0.5, 0.5], [1, 11.49999, 11.5, 11.50001, 12.5],
                                              [0, 100.5, 3.5, 180.5, 7.5], [1, 1.5, 2.5, 3.5, 4.5],
                                              [0, 254.5, 254.5, 255.5, 255.5], [1, 63.5, 127.5, 191.5, 255.5]])
    cases["offsets_push_out"] = _edit(base, trans=torch.full_like(base["trans"], 1e4) *
                                      torch.sign(torch.randn_like(base["trans"])))
    nf = make(21, n=12, C=8)
    r = nf["rois"].clone()
    vals = [float("nan"), float("inf"), -float("inf")]
    for i in range(12):
        r[i, 1 + i % 4] = vals[i % 3]
    r[0, 0] = float("nan")                           # NaN batch index truncates to 0
    t = nf["trans"].clone()
    t[::3, 0, 1, 2] = float("nan")
    t[1::3, 1, 3, 3] = float("inf")
    t[2::3, :, 0, 0] = -float("inf")
    cases["nonfinite"] = _edit(nf, rois=r.tolist(), trans=t)
    cases["no_roi"] = _edit(base, rois=torch.zeros(0, 5).tolist(), trans=torch.zeros(0, 2, 7, 7, device=DEV))
    cases["no_roi"]["rois"] = torch.zeros(0, 5, device=DEV)
    return cases


CASES = sweep() if torch.cuda.is_available() else {}
NAMES = list(CASES) or ["none"]


@pytest.mark.parametrize("no_trans", [False, True])
@pytest.mark.parametrize("name", NAMES)
def test_forward_and_count_are_the_reference_kernels_bit_for_bit(pvb, name, no_trans):
    c = CASES[name]
    ours, cnt = ours_fwd(c, no_trans)
    want, wcnt = ref_fwd(c, no_trans)
    torch.cuda.synchronize()
    assert bits_equal(cnt, wcnt), float((cnt - wcnt).abs().nan_to_num().max())
    assert bits_equal(ours, want), int((ours.view(torch.int32) != want.view(torch.int32)).sum())


GRAD_CASES = ["gradient_dpooling", "example_dpooling", "classes_4", "part_size_5", "part_size_9", "P_11_big_bins",
              "borders", "degenerate", "half_corners", "spp_8"]


def _oracle(c, no_trans):
    k = c["kw"]
    B, C, H, W = c["x"].shape
    nc = 1 if no_trans else c["trans"].shape[1] // 2
    pts = po.points(c["rois"].cpu().numpy(), c["trans"].cpu().numpy(), B, H, W, k["pooled_size"], k["part_size"],
                    k["sample_per_part"], nc, no_trans, k["spatial_scale"], k["trans_std"])
    return pts


@pytest.mark.parametrize("no_trans", [False, True])
@pytest.mark.parametrize("name", GRAD_CASES)
def test_gradients_are_within_the_rounding_bound_of_the_restatement(pvb, name, no_trans):
    """Forward and both gradients against the fp64 restatement at the kernel's own sample points: an element summed
    from m terms is within (m + a few) * u * sum |terms|.  The reference build's backward meets the same bound."""
    c = dict(CASES[name])
    if c["kw"]["trans_std"] == 0:
        c["kw"] = dict(c["kw"], trans_std=0.1)
    pts = _oracle(c, no_trans)
    x = c["x"].cpu().numpy()
    out, count, out_abs = po.forward(x, pts)
    ours, cnt = ours_fwd(c, no_trans)
    assert np.array_equal(cnt.cpu().numpy(), count)
    S = c["kw"]["sample_per_part"] ** 2
    err = np.abs(ours.double().cpu().numpy() - out)
    assert (err <= (S + 8) * U * out_abs * 1.01 + 1e-30).all(), float((err / (out_abs + 1e-30)).max())
    go = torch.randn(ours.shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    want = po.backward(x, pts, go.cpu().numpy(), c["kw"]["trans_std"])
    gi, gt = ours_bwd(c, go, no_trans)
    rgi, rgt = ref_bwd(c, go, cnt, no_trans)
    torch.cuda.synchronize()
    sides = [("ours", gi, gt), ("reference", rgi, rgt)]
    for side, a, t in sides:
        e = np.abs(a.double().cpu().numpy() - want["grad_input"])
        bound = (want["grad_input_terms"] + 6) * U * want["grad_input_abs"] * 1.01 + 1e-30
        assert (e <= bound).all(), (side, "grad_input", float((e / bound).max()))
        if no_trans:
            continue
        e = np.abs(t.double().cpu().numpy() - want["grad_trans"])
        bound = (want["grad_trans_terms"] + 10) * U * want["grad_trans_abs"] * 1.01 + 1e-30
        assert (e <= bound).all(), (side, "grad_trans", float((e / bound).max()))
    if no_trans:
        assert gt.numel() == c["trans"].numel() and not gt.any()


def test_grad_trans_is_reproducible_and_per_roi(pvb):
    c = CASES["example_dpooling"]
    go = torch.randn((20, 32, 7, 7), device=DEV)
    g1 = ours_bwd(c, go, False)[1]
    g2 = ours_bwd(c, go, False)[1]
    assert torch.equal(g1, g2)
    for i in (0, 7, 19):
        one = _edit(c, trans=c["trans"][i:i + 1])
        one["rois"] = c["rois"][i:i + 1]
        assert torch.equal(ours_bwd(one, go[i:i + 1], False)[1], g1[i:i + 1])
    big = CASES["detector_head_spp4"]
    go = torch.randn((1024, 256, 7, 7), device=DEV)
    assert torch.equal(ours_bwd(big, go, False)[1], ours_bwd(big, go, False)[1])


@pytest.mark.parametrize("no_trans", [False, True])
def test_out_of_range_batch_index_gives_zero_rows_and_no_gradient(pvb, no_trans):
    c = CASES["example_dpooling"]
    bad = torch.tensor([2, -1, 7.5, -0.5 - 1, 1e10, -1e10], device=DEV)
    rois = c["rois"].clone()
    sel = torch.arange(0, 12, 2, device=DEV)
    rois[sel, 0] = bad
    d = _edit(c)
    d["rois"] = rois
    out, cnt = ours_fwd(d, no_trans)
    keep = torch.ones(20, dtype=torch.bool, device=DEV)
    keep[sel] = False
    assert not out[sel].any() and not cnt[sel].any()
    sub = _edit(c, trans=c["trans"][keep])
    sub["rois"] = rois[keep]
    want, wcnt = ref_fwd(sub, no_trans)
    assert bits_equal(out[keep], want) and bits_equal(cnt[keep], wcnt)
    go = torch.randn_like(out)
    go_masked = go.clone()
    go_masked[sel] = 0
    gi, gt = ours_bwd(d, go, no_trans)
    _, gt0 = ours_bwd(d, go_masked, no_trans)            # the rows out of range contribute nothing
    torch.cuda.synchronize()
    if not no_trans:
        assert not gt[sel].any()
        assert torch.equal(gt[keep], gt0[keep])
    pts = _oracle(d, no_trans)
    w = po.backward(c["x"].cpu().numpy(), pts, go.cpu().numpy(), c["kw"]["trans_std"])
    e = np.abs(gi.double().cpu().numpy() - w["grad_input"])
    assert (e <= (w["grad_input_terms"] + 6) * U * w["grad_input_abs"] * 1.01 + 1e-30).all()


def test_group_size_and_bad_offsets_are_errors(pvb):
    c = CASES["example_dpooling"]
    kw = dict(c["kw"], group_size=2)
    with pytest.raises(RuntimeError, match="group_size"):
        pvb.dcn_pool.pool_forward(c["x"], c["rois"], c["trans"], no_trans=False, **kw)
    for bad in (c["trans"][:5], c["trans"][:, :1], torch.zeros(20, 2, 5, 5, device=DEV), torch.zeros(20, 6, 7, 7,
                                                                                                     device=DEV)):
        with pytest.raises(RuntimeError, match="offset must be|multiple"):
            pvb.dcn_pool.pool_forward(c["x"], c["rois"], bad, no_trans=False, **c["kw"])


def test_dcn_pooling_module_matches_the_composition_and_fills_every_gradient(pvb):
    torch.manual_seed(0)
    net = pvb.DCNPooling(1 / 4, 7, 32, False, trans_std=0.1, deform_fc_dim=64).to(DEV)
    with torch.no_grad():
        net.offset_mask_fc[4].weight.normal_(0, 0.05)
        net.offset_mask_fc[4].bias.normal_(0, 0.5)
    c = CASES["example_mdpooling"]
    x = c["x"].clone().requires_grad_()
    y = net(x, c["rois"])
    args = (1 / 4, 7, 32)
    rest = (1, 7, 4, 0.1)
    roi = pvb.dcn_v2_pooling(x, c["rois"], x.new(), *args, True, *rest)
    om = net.offset_mask_fc(roi.view(20, -1)).view(20, 3, 7, 7)
    o1, o2, mk = torch.chunk(om, 3, dim=1)
    y2 = pvb.dcn_v2_pooling(x, c["rois"], torch.cat((o1, o2), 1), *args, False, *rest) * torch.sigmoid(mk)
    assert torch.equal(y, y2)
    go = torch.randn_like(y)
    params = [x] + list(net.parameters())
    g1 = torch.autograd.grad(y, params, go, retain_graph=True)
    g2 = torch.autograd.grad(y2, params, go)
    for a, b in zip(g1, g2):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6)
    net.zero_grad()
    (y * go).sum().backward()
    for name, p in net.named_parameters():
        assert p.grad is not None and float(p.grad.abs().sum()) > 0, name
    plain = pvb.DCNPooling(1 / 4, 7, 32, True).to(DEV)
    assert torch.equal(plain(c["x"], c["rois"]), pvb.DCNv2Pooling(1 / 4, 7, 32, True)(c["x"], c["rois"], None))


def test_no_host_sync_on_a_side_stream_and_forward_graph_capture(pvb):
    c = CASES["example_dpooling"]
    want, _ = ours_fwd(c, False)
    go = torch.randn_like(want)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda.set_sync_debug_mode("error")
        try:
            out, _ = ours_fwd(c, False)
            gi, gt = ours_bwd(c, go, False)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    s.synchronize()
    assert torch.equal(out, want) and torch.isfinite(gi).all() and torch.isfinite(gt).all()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap, _ = ours_fwd(c, False)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(cap, want)


def test_empty_calls_zero_fill_the_gradients(pvb):
    c = CASES["no_roi"]
    out, cnt = ours_fwd(c, False)
    assert out.shape == (0, 32, 7, 7)
    gi, gt = ours_bwd(c, torch.zeros_like(out), False)
    torch.cuda.synchronize()
    assert gi.shape == c["x"].shape and not gi.any() and gt.shape == (0, 2, 7, 7)
    e = make(22, B=1, n=5)
    e["x"] = torch.zeros(0, 32, 64, 64, device=DEV)       # B = 0: every batch index is out of range
    out, cnt = ours_fwd(e, False)
    gi, gt = ours_bwd(e, torch.randn_like(out), False)
    torch.cuda.synchronize()
    assert not out.any() and not cnt.any() and gi.numel() == 0 and gt.shape == e["trans"].shape and not gt.any()
