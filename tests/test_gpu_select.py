"""GPU: pixel selection (csrc/select.cu: mask_bits / seg_bits -> thin_gather) against the CPU oracle's selection
(oracle/pvnet_oracle.c, orc_select_pixels), image by image.

Bar, for every image of every call: fgsum, nz, tn and state exact; xy[:tn] = (pix % W, pix // W) and dirs[:, :tn] = the
vertex at those pixels (gathered on the host) bit for bit.  The expectation of the mask-value cases is the oracle applied
to `mask.cpu().byte().long()` (v3) or `(mask == 1).long()` (distribution op): torch's own conversions."""
import numpy as np
import pytest
import torch

from util import bits_equal

pytestmark = pytest.mark.gpu

V3, DIST = 0, 1


def _run(pvb, op, mask, vertex, hn=16, **kw):
    """One call of the v3 (op 0) or distribution (op 1) operator with debug=True; returns its debug dict."""
    if op == V3:
        return pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=0.99, debug=True, **kw)[1]
    mean = torch.zeros((vertex.shape[0], vertex.shape[3], 2), device="cuda")
    return pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=hn, min_hyp_num=hn, debug=True,
                                                      **kw)[2]


def _expected(oracle, mask, op, selection=None, **kw):
    m = mask.cpu()
    m = m.byte().long() if op == V3 else (m == 1).long()
    sel = None if selection is None else selection.cpu().numpy()
    return oracle.select_pixels(m.numpy(), op, selection=sel, **kw)


def _check(dbg, want, vh, W):
    """dbg: the op's debug dict; want: oracle.select_pixels; vh: the vertex values, host numpy [B,H,W,K,2]."""
    B, K = vh.shape[0], vh.shape[3]
    skipped = want["tn"] < 0
    assert np.array_equal(dbg["fgsum"].cpu().numpy(), want["fg"])
    assert np.array_equal(dbg["nz"].cpu().numpy(), want["nz"])
    assert np.array_equal(dbg["state"].cpu().numpy(), skipped.astype(np.int32))
    assert np.array_equal(dbg["tn"].cpu().numpy(), np.where(skipped, 0, want["tn"]))
    for b in range(B):
        pix = want["pix"][b].astype(np.int64)
        t = len(pix)
        if t == 0:
            continue
        xy = np.stack([pix % W, pix // W], axis=1).astype(np.float32)
        assert bits_equal(dbg["xy"][b, :t].cpu().numpy(), xy), b
        dirs = vh[b].reshape(-1, K, 2)[pix].transpose(1, 0, 2)                 # [K,t,2]
        assert bits_equal(dbg["dirs"][b, :, :t].cpu().numpy(), dirs), b


def _planar(vertex):
    """The same values as the permuted view of a contiguous [B,2K,H,W] tensor (what decode_keypoint passes)."""
    B, H, W, K, _ = vertex.shape
    return vertex.reshape(B, H, W, 2 * K).permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1).view(B, H, W, K, 2)


# ---- 1. every BASELINE shape, whole batch, one call per (op, thinning) -------------------------------------------------
SHAPES = {
    "cfg2": ("cfg2", 16, 512),
    "cfg3": ("cfg3", 64, 1024),
    "cfg4": ("cfg4", 16, 512),
    "cfg5": (dict(B=256, H=640, W=640, K=4, hn=128, fill=(0.01, 0.80), kind="blob"), 256, 128),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_full_batch_selection_matches_oracle(pvb, oracle, shape):
    """Every image of the whole batch: v3 and the distribution op, each with the philox stream (tags 2 / 4) and with
    explicit `selection` draws, on interleaved and planar vertex layouts.  Thousands of look-back CTAs at cfg-5; cfg-4's
    12 150 bitmap words leave the last look-back block partial and rows straddle words."""
    from clean_pvnet_b200 import synth
    cfg, B, hn = SHAPES[shape]
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=1300 + len(shape) * B, B=B)
    _, H, W, K, _ = vertex.shape
    vh = vertex.cpu().numpy()
    planar = _planar(vertex)
    g = torch.Generator(device="cuda").manual_seed(B)
    selection = torch.rand((B, H, W), generator=g, device="cuda")
    fg = None
    for op, sel, vert in ((V3, None, vertex), (V3, selection, planar), (DIST, None, planar), (DIST, selection, vertex)):
        seed = 9000 + 10 * op + (sel is not None)
        dbg = _run(pvb, op, mask, vert, hn=hn if op == V3 else 64, selection=sel, seed=seed)
        want = _expected(oracle, mask, op, sel, seed=seed)
        _check(dbg, want, vh, W)
        fg = want["fg"]
        del dbg
    if shape in ("cfg3", "cfg5"):
        assert (fg > 30000).sum() >= 2 and (fg <= 30000).sum() >= 2      # thinned and unthinned images in one batch
    else:
        assert (fg > 30000).all()


# ---- 2. mask values x dtypes x load path ------------------------------------------------------------------------------
_FLOATS = [0.0, 0.0, 0.0, 1.0, 1.0, 2.0, 0.5, 0.999, 1.5, 255.7, 256.0, 257.0, -0.5, -1.0]
VALUES = {
    torch.int64: [0, 0, 0, 1, 1, 2, 255, 256, 257, -1, -255, 2 ** 32 + 1],
    torch.int32: [0, 0, 0, 1, 1, 2, 255, 256, 257, -1, -255, 65537, 2 ** 31 - 1, -2 ** 31],
    torch.int16: [0, 0, 0, 1, 1, 2, 255, 256, 257, -1, -255, 32767, -32768],
    torch.int8: [0, 0, 0, 1, 1, 2, -1, -128, 127],
    torch.uint8: [0, 0, 0, 1, 1, 2, 128, 255],
    torch.bool: [0, 0, 1],
    torch.float32: _FLOATS,
    torch.float64: _FLOATS,
    torch.float16: _FLOATS,
    torch.bfloat16: _FLOATS,
}


def _value_mask(dtype, B, H, W, seed):
    vals = torch.tensor(VALUES[dtype], dtype=torch.float64 if dtype.is_floating_point else torch.int64)
    g = torch.Generator().manual_seed(seed)
    m = vals[torch.randint(0, len(vals), (B, H, W), generator=g)].to(dtype)
    m[0, : H // 2] = 0                                    # image 0 lighter than image 1: thinned in one mode, not the other
    return m.cuda()


@pytest.mark.parametrize("dtype", list(VALUES), ids=lambda d: str(d).split(".")[-1])
def test_mask_values_every_dtype_and_load_path(pvb, oracle, dtype):
    """Foreground predicate and fg sum per dtype, through the vectorised load (contiguous, 16-byte aligned base, H*W a
    multiple of 1024) and the scalar loads (strided view; storage offset that misaligns the base; a partial last word)."""
    B, K = 2, 2
    H, W = 32, 64                                                   # 2048 pixels: two full warps of the vector path
    g = torch.Generator(device="cuda").manual_seed(7)
    base = _value_mask(dtype, B, H, W, 11)
    wide = torch.zeros((B, H, 2 * W), dtype=dtype, device="cuda")
    wide[:, :, ::2] = base
    flat = torch.zeros(B * H * W + 1, dtype=dtype, device="cuda")
    flat[1:] = base.reshape(-1)
    odd = _value_mask(dtype, B, 37, 53, 12)                        # 1961 pixels: ends inside a bitmap word
    cases = {
        "vector": base,
        "strided": wide[:, :, ::2],
        "misaligned": flat[1:].view(B, H, W),
        "partial_word": odd,
    }
    assert base.data_ptr() % 16 == 0 and not cases["strided"].is_contiguous()
    assert cases["misaligned"].is_contiguous() and cases["misaligned"].data_ptr() % 16 != 0
    for name, m in cases.items():
        vertex = torch.randn((B,) + tuple(m.shape[1:]) + (K, 2), generator=g, device="cuda")
        vh = vertex.cpu().numpy()
        for op in (V3, DIST):
            for max_num in (400, 30000):
                dbg = _run(pvb, op, m, vertex, max_num=max_num, seed=3 + op)
                want = _expected(oracle, m, op, max_num=max_num, seed=3 + op)
                assert want["tn"][1] > 0, (name, op)
                _check(dbg, want, vh, m.shape[2])


# ---- 3. boundaries ---------------------------------------------------------------------------------------------------
def _differing_fg(max_num, lo, hi):
    """Some fg in [lo, hi) whose torch ratio max_num / fg.float() differs from the correctly rounded fp32 quotient."""
    for fg in range(lo, hi):
        if np.float32(max_num) / np.float32(fg) != (max_num / torch.tensor(fg).float()).item():
            return fg
    raise AssertionError("no such fg")


def test_selection_boundaries(pvb, oracle):
    """fg == max_num (no thinning) and max_num + 1 (thinning); byte values with fgsum > max_num but nz < max_num (still
    thinned); fg == min_num (kept) and min_num - 1 (skipped); explicit draws equal to the fp32 ratio (dropped), one ulp
    below it (kept) and 0 (kept), at an fg where torch's ratio is not the correctly rounded quotient; a selection that
    drops every pixel (tn == 0 without a skip: v3 returns zeros, the distribution op NaN covariances, like the oracle)."""
    B, H, W, K = 7, 32, 64, 3
    max_num, min_num = 600, 5
    fgd = _differing_fg(max_num, 900, 1400)
    counts = [max_num, max_num + 1, 450, min_num, min_num - 1, fgd, 1000]
    g = torch.Generator().manual_seed(5)
    mask = torch.zeros((B, H * W), dtype=torch.int64)
    for b, n in enumerate(counts):
        mask[b, torch.randperm(H * W, generator=g)[:n]] = 1
    mask[2][mask[2] != 0] = 2                                      # fgsum 900 > max_num, nz 450 < max_num
    mask = mask.view(B, H, W)
    sel = torch.rand((B, H, W), generator=g)
    ratio = (max_num / torch.tensor(fgd).float()).item()
    on = torch.nonzero(mask[5].reshape(-1))[:, 0]
    s5 = sel[5].reshape(-1)
    s5[on[0::4]] = ratio                                                        # dropped
    s5[on[1::4]] = float(np.nextafter(np.float32(ratio), np.float32(0)))        # kept
    s5[on[2::8]] = 0.0                                                          # kept
    s5[on[3::8]] = float(np.float32(max_num) / np.float32(fgd))                 # the correctly rounded quotient
    sel[1].view(-1)[torch.nonzero(mask[1].reshape(-1))[0, 0]] = 0.99999          # at least one pixel of fg = max_num + 1 goes
    sel[6] = 0.99999                                                            # drops everything
    mask, sel = mask.cuda(), sel.cuda()
    vertex = torch.randn((B, H, W, K, 2), generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    vh = vertex.cpu().numpy()
    kw = dict(min_num=min_num, max_num=max_num)
    for op in (V3, DIST):
        for s in (None, sel):
            dbg = _run(pvb, op, mask, vertex, selection=s, seed=77, **kw)
            want = _expected(oracle, mask, op, s, seed=77, **kw)
            _check(dbg, want, vh, W)
            tn, nz = want["tn"], want["nz"]
            assert tn[0] == nz[0] == max_num and tn[3] == min_num and tn[4] == -1
            if op == V3:
                assert want["fg"][2] == 900 and nz[2] == 450
            if s is not None:
                kept = int((s5[on] < ratio).sum())
                assert tn[1] < nz[1] and tn[5] == kept and tn[6] == 0
                if op == V3:
                    assert tn[2] < nz[2]
    # tn == 0 without a skip: what the operators return for image 6, next to the oracle's operators
    m, v = mask.cpu().numpy(), vh
    out = pvb.ransac_voting_layer_v3(mask, vertex, 16, inlier_thresh=0.99, selection=sel, seed=1, **kw)
    want = oracle.ransac_voting_layer_v3(m, v, 16, inlier_thresh=0.99, selection=sel.cpu().numpy(), seed=1, **kw)
    assert (out[6] == 0).all() and (want[6] == 0).all()
    mean = torch.full((B, K, 2), 3.0, device="cuda")
    _, cov = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, 16, 16, selection=sel, seed=1, **kw)
    _, wcov = oracle.estimate_voting_distribution_with_mean(m, v, mean.cpu().numpy(), 16, 16, selection=sel.cpu().numpy(),
                                                            seed=1, **kw)
    assert torch.isnan(cov[6]).all() and np.isnan(wcov[6]).all()
    assert torch.isfinite(cov[:6]).all()


# ---- 4. fused decode at full size --------------------------------------------------------------------------------------
@pytest.mark.parametrize("classes", [2, 3])
@pytest.mark.parametrize("un_pnp", [False, True])
def test_fused_decode_full_size(pvb, classes, un_pnp):
    """decode_keypoint's fused argmax front end (seg_bits_kernel) at the cfg-2 shape: mask, kpt_2d and var bit-equal to
    torch.argmax + the unfused operators, whose selection the tests above pin."""
    from clean_pvnet_b200 import synth
    mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=1400 + classes, layout="planar")
    B, H, W, K, _ = vertex.shape
    g = torch.Generator(device="cuda").manual_seed(classes)
    seg = torch.randn((B, classes, H, W), generator=g, device="cuda") * 0.3
    seg[:, 1] += (mask.float() * 2 - 1) * 1.5
    ver = vertex.permute(0, 3, 4, 1, 2).reshape(B, 2 * K, H, W).contiguous()
    a = pvb.decode_keypoint({"seg": seg, "vertex": ver}, un_pnp=un_pnp, seed=21, fused=True)
    b = pvb.decode_keypoint({"seg": seg, "vertex": ver}, un_pnp=un_pnp, seed=21, fused=False)
    assert torch.equal(a["mask"], torch.argmax(seg, 1)) and torch.equal(a["mask"], b["mask"])
    if classes == 3:
        assert (a["mask"] == 2).any()                   # byte value 2: foreground for v3, not for the distribution op
    assert torch.equal(a["kpt_2d"], b["kpt_2d"])
    if un_pnp:
        assert torch.equal(a["var"], b["var"])
