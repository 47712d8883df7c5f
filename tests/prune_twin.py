"""numpy twin of the pruned v3 vote (csrc/prune.cu, DESIGN.md 4.2), in float32 like the kernels.

The one statement in Python of the cell records, the count bound, the two pass lengths and when pruning applies.
tests/test_prune_bound.py checks the bound against the oracle's exact counts on the CPU; tests/test_gpu_prune.py checks
the kernels' records against it bit for bit."""
import math

import numpy as np

CELL = 32                        # PRUNE_CELL (csrc/kernels.h)
NBIN = 128                       # PRUNE_NBIN
REC = 4 + NBIN // 2              # PRUNE_REC: box (4 floats), then 16-bit inclusive prefix counts
PASS1 = 128                      # PRUNE_M
MAX_HN = 2048                    # PRUNE_MAX_HN
MIN_UNITS = 32                   # PRUNE_MIN_UNITS
EPS = np.float32(1e-5)
F = np.float32


def prune_rotation(t):
    """prune_setup: (cos, sin) of theta' rounded outward, or None where nothing can be pruned."""
    t = float(np.float32(t))
    if not (0.0 < t < 1.0):
        return None
    w = math.acos(max(-1.0, t - 64.0 * 2.0 ** -24)) + 1e-5
    if not w < 1.5:
        return None
    return np.nextafter(F(math.cos(w)), F(0)), np.nextafter(F(math.sin(w)), F(1))


def prune_applies(t, hn, B, K):
    """prune_setup's gate, condition by condition in its order: whether the pruned vote runs for threshold t, hn
    hypotheses and B x K (image, keypoint) pairs."""
    t = float(np.float32(t))
    return (0.0 < t < 1.0 and PASS1 < hn <= MAX_HN
            and B * K >= MIN_UNITS
            and K * ((hn + 63) // 64) <= 65535           # grid.y of pass 2's 64-hypothesis slices
            and prune_rotation(t) is not None)           # theta' < 1.5


def pseudo_angle(x, y):
    """pseudo_angle (csrc/prune.cu) with IEEE division"""
    x, y = np.asarray(x, F), np.asarray(y, F)
    with np.errstate(all="ignore"):
        p = np.where(y >= 0, np.where(x >= 0, y / (x + y), F(1) + (-x) / (y - x)),
                     np.where(x < 0, F(2) + (-y) / (-x - y), F(3) + x / (x - y)))
    return p.astype(F)


def cell_records(xy, dirs, H, W):
    """prune_hist_kernel for one (image, keypoint): int32 [ceil(H/32) * ceil(W/32), REC], the words the kernel writes.
    Only pixels the reference can let vote (finite norm1 above 1e-6) enter a cell's box and histogram."""
    ncx = (W + CELL - 1) // CELL
    ncells = (H + CELL - 1) // CELL * ncx
    vx, vy = dirs[:, 0].astype(F), dirs[:, 1].astype(F)
    with np.errstate(all="ignore"):
        n1 = np.sqrt((vx.astype(np.float64) * vx + (vy * vy).astype(np.float64)).astype(F))
    ok = (n1 > F(1e-6)) & (n1 < np.inf)
    c = xy[ok].astype(F)
    cell = (c[:, 1].astype(np.int64) // CELL) * ncx + c[:, 0].astype(np.int64) // CELL
    bins = np.minimum(NBIN - 1, (pseudo_angle(vx[ok], vy[ok]) * F(NBIN // 4)).astype(np.int64))
    hist = np.zeros((ncells, NBIN), np.int64)
    np.add.at(hist, (cell, bins), 1)
    box = np.tile(np.array([np.inf, -np.inf, np.inf, -np.inf], F), (ncells, 1))
    np.minimum.at(box[:, 0], cell, c[:, 0])
    np.maximum.at(box[:, 1], cell, c[:, 0])
    np.minimum.at(box[:, 2], cell, c[:, 1])
    np.maximum.at(box[:, 3], cell, c[:, 1])
    rec = np.empty((ncells, REC), np.int32)
    rec[:, :4] = box.view(np.int32)
    rec[:, 4:] = np.cumsum(hist, 1).astype("<u2").view(np.int32)
    return rec


def count_bound(hyp, rec, tn, rot):
    """prune_bound_kernel for every hypothesis [hn,2]; tn for all when rot is None (nothing pruned)"""
    if rot is None:
        return np.full(len(hyp), tn, np.int64)
    hx, hy = hyp[:, 0].astype(F), hyp[:, 1].astype(F)
    c, s = rot
    out = np.zeros(len(hyp), np.int64)
    with np.errstate(all="ignore"):
        for r in rec:
            P = r[4:].view("<u2").astype(np.int64)
            tot = int(P[-1])
            if tot == 0:
                continue
            x0, x1, y0, y1 = r[:4].view(F)
            inside = (hx >= x0 - F(0.5)) & (hx <= x1 + F(0.5)) & (hy >= y0 - F(0.5)) & (hy <= y1 + F(0.5))
            lx, ly = hx - x0, hy - y0
            ux, uy = lx.copy(), ly.copy()
            for cx, cy in ((x1, y0), (x0, y1), (x1, y1)):
                dx, dy = hx - cx, hy - cy
                m = lx * dy - ly * dx < 0
                lx, ly = np.where(m, dx, lx), np.where(m, dy, ly)
                m = ux * dy - uy * dx > 0
                ux, uy = np.where(m, dx, ux), np.where(m, dy, uy)
            plo = pseudo_angle(c * lx + s * ly, c * ly - s * lx)
            phi = pseudo_angle(c * ux - s * uy, c * uy + s * ux)
            phi = np.where(phi < plo, phi + F(4), phi)
            blo = np.floor((plo - EPS) * F(NBIN // 4)).astype(np.int64)
            bhi = np.floor((phi + EPS) * F(NBIN // 4)).astype(np.int64)
            Pex = np.concatenate([[0], P])

            def C(j):
                w = np.floor_divide(j, NBIN)
                return Pex[j - w * NBIN] + tot * w
            part = np.where(bhi - blo + 1 >= NBIN, tot, C(bhi + 1) - C(blo))
            out += np.where(inside, tot, part)
    out[~(np.abs(hx) + np.abs(hy) <= F(1e15))] = tn
    return out


def scored(bnd, cnt):
    """Slots the two passes fill (prune_plan_kernel, then prune_next_kernel): the PASS1 largest bounds (ties in index
    order), then every other h with B(h) >= L, L the best exact count of pass 1"""
    p1 = np.argsort(-bnd, kind="stable")[:PASS1]
    rest = np.ones(len(bnd), bool)
    rest[p1] = False
    return PASS1 + int(np.count_nonzero(rest & (bnd >= cnt[p1].max())))


def field(xy, kp, rng, noise=0.02):
    """unit directions from each pixel towards kp, with angular noise (radians)"""
    d = kp[None, :] - xy
    a = np.arctan2(d[:, 1], d[:, 0]) + rng.normal(0, noise, len(xy))
    return np.stack([np.cos(a), np.sin(a)], 1).astype(F)


def near(h, rng, n):
    """points within a few ulps of h, and h itself"""
    out = [h]
    for _ in range(n):
        out.append([np.nextafter(F(h[0]), F(np.inf) if rng.random() < 0.5 else F(-np.inf)),
                    np.nextafter(F(h[1]), F(np.inf) if rng.random() < 0.5 else F(-np.inf))])
    return np.array(out, F)
