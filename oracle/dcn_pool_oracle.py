"""numpy fp64 restatement of clean-pvnet's deformable PSROI pooling (lib/csrc/dcn_v2/src/cuda/
dcn_v2_psroi_pooling_cuda.cu): the forward, the count and both gradients, with the reference's predicates and layouts.
TEST INFRASTRUCTURE ONLY.

    points(rois, trans, B, H, W, P, part_size, spp, num_classes, no_trans, spatial_scale, trans_std, exact=False)
        -> dict of the sample points [n, nc, P, P, spp*spp]: w, h (clamped), valid, and per ROI batch, roi_w, roi_h
    forward(x, pts)                        -> out, count, out_abs        [n, C, P, P]
    backward(x, pts, grad_out, trans_std)  -> dict of grad_input, grad_trans and each one's `_abs` and `_terms`

points() rounds like the sm_90a build of the reference kernel (fp32 with the fused multiply-adds its SASS shows, the
range test and clamp in fp64; DESIGN.md 8m), so forward / backward see the sample points the fp32 kernels see.  With
exact=True every step is fp64 instead, which makes the forward a smooth function of trans for finite differences.
Everything after the sample point is fp64.  Each value comes with the sum of the absolute values of its terms, so a test
can bound an fp32 result by (terms + a few) * 2^-24 * abs.  Gradients assume finite inputs.
"""
import numpy as np

F32, F64 = np.float32, np.float64


def fma32(a, b, c):
    """fp32 fma(a, b, c), rounded once: the fp64 product is exact, the fp64 sum is rounded to odd, and rounding that to
    fp32 is then correct (53 >= 24 + 2)."""
    a, b, c = (np.asarray(v, F32).astype(F64) for v in (a, b, c))
    p = a * b
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        fix = np.isfinite(s) & (e != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(F32)


def _round_half_away(x):
    with np.errstate(invalid="ignore"):
        return (np.sign(x) * np.floor(np.abs(x.astype(F64)) + 0.5)).astype(F32)


def points(rois, trans, B, H, W, P, part_size, spp, num_classes, no_trans, spatial_scale, trans_std, exact=False):
    rois = np.asarray(rois, F32).reshape(-1, 5)
    n, nc, S = rois.shape[0], (1 if no_trans else num_classes), spp * spp
    scale, std = F32(spatial_scale), F32(trans_std)
    with np.errstate(invalid="ignore", over="ignore"):
        bi = rois[:, 0]
        batch = np.where(np.isnan(bi), 0, np.trunc(np.nan_to_num(bi, nan=0, posinf=2 ** 31 - 1, neginf=-2 ** 31)))
        batch = np.clip(batch, -2 ** 31, 2 ** 31 - 1).astype(np.int64)
        x1, y1, x2, y2 = (_round_half_away(rois[:, i]) for i in (1, 2, 3, 4))
        pw = np.arange(P)
        part = np.minimum(np.floor((pw.astype(F32) / F32(P)).astype(F32) * F32(part_size)).astype(np.int64),
                          part_size - 1)
        iy, ix = np.divmod(np.arange(S), spp)
        if no_trans:
            t = np.zeros((n, nc, 2, P, P), F64 if exact else F32)
        else:
            tr = np.asarray(trans, F64 if exact else F32).reshape(n, nc, 2, part_size, part_size)
            tr = tr[:, :, :, part[:, None], part[None, :]]                    # [n, nc, 2, P(ph), P(pw)]
            t = tr.astype(F64) * F64(std) if exact else (tr * std).astype(F32)
        if exact:
            sw, sh = x1.astype(F64) * scale - 0.5, y1.astype(F64) * scale - 0.5
            rw = np.fmax((x2.astype(F64) + 1) * scale - 0.5 - sw, 0.1)
            rh = np.fmax((y2.astype(F64) + 1) * scale - 0.5 - sh, 0.1)
            bw, bh = rw / P, rh / P
            subw, subh = bw / spp, bh / spp
            ws = pw[None, None, None, :] * bw[:, None, None, None] + sw[:, None, None, None] + \
                t[:, :, 0] * rw[:, None, None, None]
            hs = pw[None, None, :, None] * bh[:, None, None, None] + sh[:, None, None, None] + \
                t[:, :, 1] * rh[:, None, None, None]
            w = ws[..., None] + ix * subw[:, None, None, None, None]
            h = hs[..., None] + iy * subh[:, None, None, None, None]
        else:
            sw, sh = fma32(x1, scale, -0.5), fma32(y1, scale, -0.5)
            ew, eh = fma32((x2 + F32(1)).astype(F32), scale, -0.5), fma32((y2 + F32(1)).astype(F32), scale, -0.5)
            rw = np.fmax((ew - sw).astype(F32).astype(F64), 0.1).astype(F32)
            rh = np.fmax((eh - sh).astype(F32).astype(F64), 0.1).astype(F32)
            bw, bh = (rw / F32(P)).astype(F32), (rh / F32(P)).astype(F32)
            subw, subh = (bw / F32(spp)).astype(F32), (bh / F32(spp)).astype(F32)
            shp = (n, nc, P, P)
            ws = fma32(t[:, :, 0], rw[:, None, None, None],
                       np.broadcast_to(fma32(pw[None, :].astype(F32), bw[:, None], sw[:, None])[:, None, None, :], shp))
            hs = fma32(t[:, :, 1], rh[:, None, None, None],
                       np.broadcast_to(fma32(pw[None, :].astype(F32), bh[:, None], sh[:, None])[:, None, :, None], shp))
            w = fma32(ix.astype(F32), subw[:, None, None, None, None], ws[..., None])
            h = fma32(iy.astype(F32), subh[:, None, None, None, None], hs[..., None])
        wd, hd = w.astype(F64), h.astype(F64)
        valid = ~((wd < -0.5) | (wd > W - 0.5) | (hd < -0.5) | (hd > H - 0.5))
        valid &= ((batch >= 0) & (batch < B))[:, None, None, None, None]
        wc, hc = np.fmin(np.fmax(wd, 0.0), W - 1.0), np.fmin(np.fmax(hd, 0.0), H - 1.0)
        if not exact:
            wc, hc = wc.astype(F32).astype(F64), hc.astype(F32).astype(F64)
    return dict(w=wc, h=hc, valid=valid, batch=batch, roi_w=np.asarray(rw, F64), roi_h=np.asarray(rh, F64), H=H, W=W,
                P=P, part_size=part_size, part=part, nc=nc)


def _corners(x, pts):
    """Per sample [n, nc, P, P, S]: the corner indices (y1, y2, x1, x2), weights q00, q01, q10, q11, dx, dy, and the
    four corner values of every channel [n, nc, cec, P, P, S] as v11, v12, v21, v22 (the reference's names)."""
    B, C, H, W = x.shape
    nc = pts["nc"]
    cec = C // nc
    ok = pts["valid"]
    w, h = np.where(ok, pts["w"], 0.0), np.where(ok, pts["h"], 0.0)
    xa, xb, ya, yb = np.floor(w).astype(np.int64), np.ceil(w).astype(np.int64), np.floor(h).astype(np.int64), \
        np.ceil(h).astype(np.int64)
    dx, dy = w - xa, h - ya
    b = np.clip(pts["batch"], 0, max(B - 1, 0))[:, None, None, None, None]
    xg = np.asarray(x, F64).reshape(B, nc, cec, H * W) if B else np.zeros((1, nc, cec, H * W))
    vals = {}
    for name, yy, xx in (("v11", ya, xa), ("v12", yb, xa), ("v21", ya, xb), ("v22", yb, xb)):
        lin = yy * W + xx                                               # [n, nc, P, P, S]
        g = xg[b[:, :, 0, 0, 0][:, 0]]                                  # [n, nc, cec, HW]
        idx = np.broadcast_to(lin.reshape(lin.shape[0], nc, 1, -1), g.shape[:3] + (lin[0, 0].size,))
        vals[name] = np.take_along_axis(g, idx, axis=3).reshape(g.shape[:3] + lin.shape[2:])
    q = dict(q00=(1 - dx) * (1 - dy), q01=(1 - dx) * dy, q10=dx * (1 - dy), q11=dx * dy)
    return (ya, yb, xa, xb), q, dx, dy, vals


def forward(x, pts):
    B, C, H, W = x.shape
    nc, P = pts["nc"], pts["P"]
    n = pts["valid"].shape[0]
    ok = pts["valid"][:, :, None]                                       # [n, nc, 1, P, P, S]
    _, q, _, _, v = _corners(x, pts)
    terms = [q["q00"][:, :, None] * v["v11"], q["q01"][:, :, None] * v["v12"], q["q10"][:, :, None] * v["v21"],
             q["q11"][:, :, None] * v["v22"]]
    cnt = pts["valid"].sum(axis=-1).astype(F64)[:, :, None]             # [n, nc, 1, P, P]
    s = np.where(ok, sum(terms), 0.0).sum(axis=-1)
    s_abs = np.where(ok, sum(np.abs(t) for t in terms), 0.0).sum(axis=-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(cnt > 0, s / np.maximum(cnt, 1), 0.0)
        out_abs = np.where(cnt > 0, s_abs / np.maximum(cnt, 1), 0.0)
    count = np.broadcast_to(cnt, out.shape)
    return out.reshape(n, C, P, P), count.reshape(n, C, P, P).copy(), out_abs.reshape(n, C, P, P)


def backward(x, pts, grad_out, trans_std):
    B, C, H, W = x.shape
    nc, P, ps = pts["nc"], pts["P"], pts["part_size"]
    n = pts["valid"].shape[0]
    cec = C // nc
    ok = pts["valid"][:, :, None]
    (ya, yb, xa, xb), q, dx, dy, v = _corners(x, pts)
    cnt = pts["valid"].sum(axis=-1).astype(F64)[:, :, None]             # [n, nc, 1, P, P]
    go = np.asarray(grad_out, F64).reshape(n, nc, cec, P, P)
    diff = np.where(cnt > 0, go / np.maximum(cnt, 1), 0.0)[..., None]   # [n, nc, cec, P, P, 1]
    r = {}
    gi, gi_abs, gi_cnt = (np.zeros(B * C * H * W) for _ in range(3))
    b = pts["batch"]
    plane = ((np.clip(b, 0, None)[:, None, None] * C + np.arange(nc)[None, :, None] * cec +
              np.arange(cec)[None, None, :]) * (H * W))[..., None, None, None]       # [n, nc, cec, 1, 1, 1]
    shp = (n, nc, cec, P, P, dx.shape[-1])
    okb = np.broadcast_to(ok, shp).ravel()
    for wq, yy, xx in ((q["q00"], ya, xa), (q["q01"], yb, xa), (q["q10"], ya, xb), (q["q11"], yb, xb)):
        lin = np.broadcast_to(plane + (yy * W + xx)[:, :, None], shp).ravel()[okb]
        term = np.broadcast_to(wq[:, :, None] * diff, shp).ravel()[okb]
        np.add.at(gi, lin, term)
        np.add.at(gi_abs, lin, np.abs(term))
        np.add.at(gi_cnt, lin, 1.0)
    r["grad_input"], r["grad_input_abs"] = gi.reshape(B, C, H, W), gi_abs.reshape(B, C, H, W)
    r["grad_input_terms"] = gi_cnt.reshape(B, C, H, W)

    # d(value)/dw and d(value)/dh with U00 = v11, U01 = v12, U10 = v21, U11 = v22 (:255-262)
    dyc, dxc = dy[:, :, None], dx[:, :, None]
    tx = [dyc * v["v22"], (1 - dyc) * v["v21"], -dyc * v["v12"], -(1 - dyc) * v["v11"]]
    ty = [dxc * v["v22"], (1 - dxc) * v["v12"], -dxc * v["v21"], -(1 - dxc) * v["v11"]]
    sx = trans_std * diff * pts["roi_w"][:, None, None, None, None, None]
    sy = trans_std * diff * pts["roi_h"][:, None, None, None, None, None]
    gx = np.where(ok, sum(tx) * sx, 0.0)
    gy = np.where(ok, sum(ty) * sy, 0.0)
    gx_abs = np.where(ok, sum(np.abs(t) for t in tx) * np.abs(sx), 0.0)
    gy_abs = np.where(ok, sum(np.abs(t) for t in ty) * np.abs(sy), 0.0)
    part = pts["part"]
    gt, gt_abs, gt_terms = (np.zeros((n, nc, 2, ps, ps)) for _ in range(3))
    for ph in range(P):
        for pw in range(P):
            cy, cx = part[ph], part[pw]
            gt[:, :, 0, cy, cx] += gx[:, :, :, ph, pw].sum(axis=(2, 3))
            gt[:, :, 1, cy, cx] += gy[:, :, :, ph, pw].sum(axis=(2, 3))
            gt_abs[:, :, 0, cy, cx] += gx_abs[:, :, :, ph, pw].sum(axis=(2, 3))
            gt_abs[:, :, 1, cy, cx] += gy_abs[:, :, :, ph, pw].sum(axis=(2, 3))
            gt_terms[:, :, :, cy, cx] += cec * pts["valid"][:, :, ph, pw].sum(axis=-1)[:, :, None]
    r["grad_trans"] = gt.reshape(n, 2 * nc, ps, ps)
    r["grad_trans_abs"] = gt_abs.reshape(n, 2 * nc, ps, ps)
    r["grad_trans_terms"] = gt_terms.reshape(n, 2 * nc, ps, ps)
    return r
