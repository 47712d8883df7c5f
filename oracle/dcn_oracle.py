"""numpy fp64 restatement of clean-pvnet's DCNv2 (lib/csrc/dcn_v2/src/cuda/dcn_v2_im2col_cuda.cu + dcn_v2_cuda.cu):
the forward and all five gradients, with the reference's predicates and layouts.   TEST INFRASTRUCTURE ONLY.

Every value comes with the sum of the absolute values of its terms (`*_abs`), so a test can bound an fp32 result by
n * 2^-24 * abs, n the longest accumulation chain.  The sample point is rounded to fp32 exactly like the reference
(h = float32(float(ho*s - p + i*d) + dy)); everything after that is fp64.

    cols(x, offset, mask, kh, kw, stride, pad, dil, dg)                 -> col, col_abs  [B, C*kh*kw, Ho*Wo]
    forward(x, offset, mask, weight, bias, stride, pad, dil, dg)        -> out, out_abs  [B, C_out, Ho, Wo]
    backward(x, offset, mask, weight, bias, grad_out, stride, pad, dil, dg)
        -> dict of grad_input, grad_offset, grad_mask, grad_weight, grad_bias, grad_cols and each one's `_abs`
stride / pad / dil are (h, w) pairs.  Gradients assume finite sample points (no NaN offsets).
"""
import numpy as np


def out_size(H, W, kh, kw, stride, pad, dil):
    return ((H + 2 * pad[0] - (dil[0] * (kh - 1) + 1)) // stride[0] + 1,
            (W + 2 * pad[1] - (dil[1] * (kw - 1) + 1)) // stride[1] + 1)


def _points(x, offset, kh, kw, stride, pad, dil, dg):
    """fp32 sample coordinates h, w [B, dg, T, Ho, Wo]."""
    B, C, H, W = x.shape
    Ho, Wo = out_size(H, W, kh, kw, stride, pad, dil)
    T = kh * kw
    off = np.asarray(offset, np.float32).reshape(B, dg, T, 2, Ho, Wo)
    ii, jj = np.divmod(np.arange(T), kw)
    bh = (np.arange(Ho)[None, :, None] * stride[0] - pad[0] + ii[:, None, None] * dil[0]).astype(np.float32)
    bw = (np.arange(Wo)[None, None, :] * stride[1] - pad[1] + jj[:, None, None] * dil[1]).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        h = (bh[None, None] + off[:, :, :, 0]).astype(np.float32)
        w = (bw[None, None] + off[:, :, :, 1]).astype(np.float32)
    return h, w


def _corners(x, h, w, dg):
    """The four corners of every sample point: value [B, dg, Cg, T, Ho, Wo] and in-image flag [B, dg, 1, T, Ho, Wo]
    of each, plus hl, wl (floors) and the fp64 coordinates."""
    B, C, H, W = x.shape
    Cg = C // dg
    hd, wd = h.astype(np.float64), w.astype(np.float64)
    with np.errstate(invalid="ignore"):
        hl = np.floor(np.nan_to_num(hd, nan=0.0, posinf=1e9, neginf=-1e9)).astype(np.int64)
        wl = np.floor(np.nan_to_num(wd, nan=0.0, posinf=1e9, neginf=-1e9)).astype(np.int64)
    xg = np.asarray(x, np.float64).reshape(B, dg, Cg, H * W)
    vals, inside = [], []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        yy, xx = hl + dy, wl + dx
        ok = (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
        idx = np.where(ok, yy * W + xx, 0).reshape(B, dg, 1, -1)
        v = np.take_along_axis(xg, np.broadcast_to(idx, (B, dg, Cg, idx.shape[-1])), axis=3)
        v = v.reshape((B, dg, Cg) + h.shape[2:]) * ok[:, :, None]
        vals.append(v)
        inside.append(ok[:, :, None])
    return vals, inside, hl[:, :, None], wl[:, :, None], hd[:, :, None], wd[:, :, None]


def cols(x, offset, mask, kh, kw, stride, pad, dil, dg):
    B, C, H, W = x.shape
    h, w = _points(x, offset, kh, kw, stride, pad, dil, dg)
    T = kh * kw
    m = np.asarray(mask, np.float64).reshape((B, dg, 1) + h.shape[2:])
    with np.errstate(invalid="ignore"):
        used = ((h > -1) & (w > -1) & (h < H) & (w < W))[:, :, None]
    (v1, v2, v3, v4), _, hl, wl, hd, wd = _corners(x, h, w, dg)
    lh, lw = np.where(used, hd - hl, 0.0), np.where(used, wd - wl, 0.0)
    hh, hw = 1 - lh, 1 - lw
    terms = [hh * hw * v1, hh * lw * v2, lh * hw * v3, lh * lw * v4]
    val = np.where(used, sum(terms), 0.0)
    val_abs = np.where(used, sum(np.abs(t) for t in terms), 0.0)
    col = (val * m).reshape(B, C * T, -1)
    col_abs = (val_abs * np.abs(m)).reshape(B, C * T, -1)
    return col, col_abs


def forward(x, offset, mask, weight, bias, stride, pad, dil, dg):
    Co, C, kh, kw = weight.shape
    B, _, H, W = x.shape
    Ho, Wo = out_size(H, W, kh, kw, stride, pad, dil)
    col, col_abs = cols(x, offset, mask, kh, kw, stride, pad, dil, dg)
    W2 = np.asarray(weight, np.float64).reshape(Co, -1)
    b = np.asarray(bias, np.float64)[None, :, None]
    out = b + np.einsum("ok,bkp->bop", W2, col)
    out_abs = np.abs(b) + np.einsum("ok,bkp->bop", np.abs(W2), col_abs)
    return out.reshape(B, Co, Ho, Wo), out_abs.reshape(B, Co, Ho, Wo)


def backward(x, offset, mask, weight, bias, grad_out, stride, pad, dil, dg):
    Co, C, kh, kw = weight.shape
    B, _, H, W = x.shape
    Ho, Wo = out_size(H, W, kh, kw, stride, pad, dil)
    T, Cg, P = kh * kw, C // dg, Ho * Wo
    W2 = np.asarray(weight, np.float64).reshape(Co, -1)
    go = np.asarray(grad_out, np.float64).reshape(B, Co, P)
    r = {}
    gc = np.einsum("ok,bop->bkp", W2, go)
    gc_abs = np.einsum("ok,bop->bkp", np.abs(W2), np.abs(go))
    r["grad_cols"], r["grad_cols_abs"] = gc, gc_abs
    col, col_abs = cols(x, offset, mask, kh, kw, stride, pad, dil, dg)
    r["grad_weight"] = np.einsum("bop,bkp->ok", go, col).reshape(weight.shape)
    r["grad_weight_abs"] = np.einsum("bop,bkp->ok", np.abs(go), col_abs).reshape(weight.shape)
    r["grad_bias"], r["grad_bias_abs"] = go.sum(axis=(0, 2)), np.abs(go).sum(axis=(0, 2))

    h, w = _points(x, offset, kh, kw, stride, pad, dil, dg)
    shp = (B, dg, Cg, T, Ho, Wo)
    g5, g5_abs = gc.reshape(shp), gc_abs.reshape(shp)
    m = np.asarray(mask, np.float64).reshape((B, dg, 1, T, Ho, Wo))
    (v1, v2, v3, v4), _, hl, wl, hd, wd = _corners(x, h, w, dg)
    # col2im_coord: a point with h <= -1, w <= -1, h >= H or w >= W contributes 0
    dom = ~((h <= -1) | (w <= -1) | (h >= H) | (w >= W))[:, :, None]
    lh, lw = hd - hl, wd - wl
    hh, hw = 1 - lh, 1 - lw
    vt = [hh * hw * v1, hh * lw * v2, lh * hw * v3, lh * lw * v4]
    val, val_abs = sum(vt), sum(np.abs(t) for t in vt)
    gm = np.where(dom, g5 * val, 0.0).sum(axis=2)
    gm_abs = np.where(dom, g5_abs * val_abs, 0.0).sum(axis=2)
    ty = [-hw * v1, -lw * v2, hw * v3, lw * v4]        # d(value)/dh
    tx = [-hh * v1, hh * v2, -lh * v3, lh * v4]        # d(value)/dw
    gy = np.where(dom, sum(ty) * g5 * m, 0.0).sum(axis=2)
    gx = np.where(dom, sum(tx) * g5 * m, 0.0).sum(axis=2)
    gy_abs = np.where(dom, sum(np.abs(t) for t in ty) * g5_abs * np.abs(m), 0.0).sum(axis=2)
    gx_abs = np.where(dom, sum(np.abs(t) for t in tx) * g5_abs * np.abs(m), 0.0).sum(axis=2)
    r["grad_mask"] = gm.reshape(B, dg * T, Ho, Wo)
    r["grad_mask_abs"] = gm_abs.reshape(B, dg * T, Ho, Wo)
    r["grad_offset"] = np.stack([gy, gx], axis=3).reshape(B, dg * 2 * T, Ho, Wo)
    r["grad_offset_abs"] = np.stack([gy_abs, gx_abs], axis=3).reshape(B, dg * 2 * T, Ho, Wo)

    # col2im: the used sample points scatter their bilinear weights; the high corner only when h > floor(h)
    used = ((h > -1) & (w > -1) & (h < H) & (w < W))[:, :, None]
    gi, gi_abs, gi_cnt = np.zeros(B * C * H * W), np.zeros(B * C * H * W), np.zeros(B * C * H * W)
    top, top_abs = g5 * m, g5_abs * np.abs(m)
    plane = (np.arange(B * dg * Cg) * (H * W)).reshape(B, dg, Cg, 1, 1, 1)
    for dy, dx, wt in ((0, 0, hh * hw), (0, 1, hh * lw), (1, 0, lh * hw), (1, 1, lh * lw)):
        yy, xx = hl + dy, wl + dx
        ok = used & (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        if dy:
            ok &= hd > hl
        if dx:
            ok &= wd > wl
        lin = np.broadcast_to(plane + np.where(ok, yy * W + xx, 0), shp).ravel()
        okb = np.broadcast_to(ok, shp).ravel()
        np.add.at(gi, lin[okb], np.broadcast_to(wt * top, shp).ravel()[okb])
        np.add.at(gi_abs, lin[okb], np.broadcast_to(np.abs(wt) * top_abs, shp).ravel()[okb])
        np.add.at(gi_cnt, lin[okb], 1.0)
    r["grad_input"] = gi.reshape(B, C, H, W)
    r["grad_input_abs"] = gi_abs.reshape(B, C, H, W)
    r["grad_input_terms"] = gi_cnt.reshape(B, C, H, W)
    return r
