"""numpy model of pass 1's per-box classification (DESIGN.md 4.2, "Pass 1 per box of hypotheses"), in float32 like the
vote kernel's fast path.

For one tile of selected pixels and a box H around some of pass 1's hypotheses (in the tile frame of the fast path) each
pixel is a certain inlier (the margin exceeds the box's guard band at all four corners), a certain outlier (L+ or L-
is below minus the band at all four corners) or uncertain.  Only uncertain pixels are scored one hypothesis at a time.
tests/test_pass1_boxes_host.py checks the classification against the oracle's exact verdicts on the CPU;
`python tests/pass1_box_twin.py` reports the share of certain pixels on the bench workloads and the instruction count it
predicts for pass 1 with each way of forming boxes."""
import math
import os
import sys

import numpy as np

F = np.float32
TILE = 1024                     # pass 1's pixels per CTA (vote_kernel<4,128,8,1024,1>)
PASS1 = 128                     # PRUNE_M
TEST_INSTR = 7.1                # instructions per scored test (DESIGN.md 4.1)
CLASSIFY_INSTR = 40             # per (pixel, box): 12 FFMA, 8 FADD, the minima, 3 compares, the compaction


def cone_params(t):
    """make_cone (csrc/vote.cu): (kappa, band, floor) in float32"""
    t = float(F(t))
    s = math.sqrt(1.0 - t * t)
    kappa, G = s / t, 1.0 / (t * s)
    band = 1.25 * 2.0 ** -24 * (18.0 + 22.0 * kappa + 9.0 * G)
    return F(kappa), np.nextafter(F(band), F(np.inf)), np.nextafter(F(2e-6 * (kappa + 1.0)), F(np.inf))


def tile_records(xy, dirs, kappa):
    """load_tile + cone_record for one tile: records [n, 6] (A1, A2, A3, B1, B2, B3) and the origin (ox, oy, cmax).
    Pixels the reference never lets vote get A3 = -1e30, pixels outside the analysed domain all zeros."""
    xy, dirs = xy.astype(F), dirs.astype(F)
    x0, x1, y0, y1 = xy[:, 0].min(), xy[:, 0].max(), xy[:, 1].min(), xy[:, 1].max()
    ox, oy = F(0.5) * (x0 + x1), F(0.5) * (y0 + y1)
    cmax = (F(0.5) * (x1 - x0) + F(0.5) * (y1 - y0)) * F(1.000001) + F(1e-3)
    vx, vy = dirs[:, 0], dirs[:, 1]
    rec = np.zeros((len(xy), 6), F)
    rec[:, 2] = F(-1e30)
    with np.errstate(all="ignore"):
        n1 = np.sqrt(vx * vx + vy * vy)
        cxc, cyc = xy[:, 0] - ox, xy[:, 1] - oy
        vote = n1 > F(1e-6)
        out = vote & ~((n1 < F(1e18)) & (np.abs(cxc) + np.abs(cyc) <= cmax))
        ok = vote & ~out
        ux, uy = vx / n1, vy / n1
        a1, a2 = kappa * ux, kappa * uy
    rec[out] = 0
    rec[ok, 0], rec[ok, 1], rec[ok, 2] = a1[ok], a2[ok], -(a1[ok] * cxc[ok] + a2[ok] * cyc[ok])
    rec[ok, 3], rec[ok, 4], rec[ok, 5] = -uy[ok], ux[ok], uy[ok] * cxc[ok] - ux[ok] * cyc[ok]
    return rec, ox, oy, cmax


def hyp_frame(hyp, ox, oy):
    """hyp_frame's tile-frame coordinates, and whether the hypothesis is finite and not huge (its band is finite)"""
    with np.errstate(all="ignore"):
        xc, yc = hyp[:, 0].astype(F) - ox, hyp[:, 1].astype(F) - oy
        ok = np.abs(xc) + np.abs(yc) <= F(1e15)
    return xc, yc, ok


def classify(rec, xc, yc, ok, cmax, band, floor):
    """Per pixel of the tile: +1 certain inlier, -1 certain outlier, 0 uncertain, for the box around the tile-frame
    points (xc, yc); a box holding an unbounded hypothesis leaves every pixel uncertain"""
    if not ok.all():
        return np.zeros(len(rec), np.int8)
    X, Y = (xc.min(), xc.max()), (yc.min(), yc.max())
    smax = max(abs(x) + abs(y) for x in X for y in Y) + cmax
    d = max(band * smax, floor)
    a, p = [], []
    for x in X:
        for y in Y:
            a.append(rec[:, 0] * x + (rec[:, 1] * y + rec[:, 2]))
            p.append(rec[:, 3] * x + (rec[:, 4] * y + rec[:, 5]))
    a, p = np.array(a), np.array(p)
    inlier = ((a - np.abs(p)) > d).all(0)
    outlier = ((a + p) < -d).all(0) | ((a - p) < -d).all(0)
    return np.where(inlier, 1, np.where(outlier, -1, 0)).astype(np.int8)


def boxes(xc, yc, size):
    """Pass 1's hypotheses in groups of `size`: kd-order (halve by the wider extent, recursively), a deterministic
    spatial sort"""
    idx = np.arange(len(xc))

    def split(ix):
        if len(ix) <= size:
            return [ix]
        x, y = xc[ix], yc[ix]
        key = x if np.ptp(x) >= np.ptp(y) else y
        o = ix[np.argsort(key, kind="stable")]
        h = len(o) // 2
        return split(o[:h]) + split(o[h:])
    return split(idx)


def pair_stats(xy, dirs, hyp, t, sizes=(128, 32, 16)):
    """For one (image, keypoint) and pass 1's hypotheses: {box size: (certain pixel-box pairs, pixel-box pairs,
    predicted instructions)} summed over the tiles, and the instructions of today's per-hypothesis scoring"""
    kappa, band, floor = cone_params(t)
    out = {s: np.zeros(3) for s in sizes}
    today = 0.0
    for t0 in range(0, len(xy), TILE):
        rec, ox, oy, cmax = tile_records(xy[t0:t0 + TILE], dirs[t0:t0 + TILE], kappa)
        xc, yc, ok = hyp_frame(hyp, ox, oy)
        today += len(rec) * len(hyp) * TEST_INSTR
        for s in sizes:
            for g in boxes(xc, yc, s):
                c = classify(rec, xc[g], yc[g], ok[g], cmax, band, floor)
                nu = np.count_nonzero(c == 0)
                out[s] += (len(rec) - nu, len(rec), len(rec) * CLASSIFY_INSTR + nu * len(g) * TEST_INSTR)
    return out, today


def workload_report(cfg, seeds, B=None, t=0.99, sizes=(128, 32, 16)):
    """The model's totals over every (image, keypoint) of `cfg` for the given seeds"""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    import pvnet_oracle as po
    from prune_twin import cell_records, count_bound, prune_rotation
    from clean_pvnet_b200 import synth
    tot = {s: np.zeros(3) for s in sizes}
    today = 0.0
    for seed in seeds:
        mask, vertex, _ = synth.make_inputs(cfg, device="cpu", seed=seed, B=B)
        m, v = mask.numpy(), vertex.numpy()
        _, dbg = po.ransac_voting_layer_v3(m, v, 512, inlier_thresh=t, seed=seed, debug=True)
        sel = po.select_pixels(m, mode=0, seed=seed)
        H, W = m.shape[1:]
        for b in range(m.shape[0]):
            pix = sel["pix"][b]
            xy = np.stack([pix % W, pix // W], 1).astype(F)
            for k in range(v.shape[3]):
                d = v[b, pix // W, pix % W, k].astype(F)
                hyp = dbg["hyp"][b, k].astype(F)
                bnd = count_bound(hyp, cell_records(xy, d, H, W), len(pix), prune_rotation(t))
                p1 = np.sort(np.argsort(-bnd, kind="stable")[:PASS1])
                st, td = pair_stats(xy, d, hyp[p1], t, sizes)
                today += td
                for s in sizes:
                    tot[s] += st[s]
    return tot, today


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    for cfg, B in (("cfg2", None), ("cfg4", 4)):
        tot, today = workload_report(cfg, (1236, 1237, 1238), B=B)
        print(f"{cfg} (B = {B or 16}, seeds 1236-1238, t = 0.99): pass 1 today {today / 1e9:.3f} G instructions")
        for s, (cert, pairs, ins) in tot.items():
            print(f"  boxes of {s:3d}: certain {cert / pairs:6.1%} of pixel-box pairs, "
                  f"{ins / 1e9:.3f} G instructions, {today / ins:.2f}x fewer")


if __name__ == "__main__":
    main()
