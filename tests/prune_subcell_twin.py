"""numpy twin of the pruned v3 vote's 16x16-pixel sub-cell records and its two pass lists (csrc/prune.cu, DESIGN.md 4.2),
in float32 like the kernels; the cell records, the count bound and the gate are prune_twin's.

tests/test_prune_subcell.py checks the bound over these records against the oracle's exact counts on the CPU;
tests/test_gpu_prune_subcell.py checks the kernels' sub-cell records against them bit for bit."""
import numpy as np

from prune_twin import CELL, F, NBIN, PASS1, REC, pseudo_angle

SUB = 16                         # PRUNE_SUB (csrc/kernels.h)


def subcell_records(xy, dirs, H, W):
    """prune_hist_kernel's sub-cell records for one (image, keypoint): int32 [ncells, 4, REC], the 16x16-pixel quarters
    of each 32x32 cell (top left, top right, bottom left, bottom right), empty where they lie outside the image.  Only
    pixels the reference can let vote (finite norm1 above 1e-6) enter a box and histogram, as in cell_records."""
    ncx = (W + CELL - 1) // CELL
    nsub = (H + CELL - 1) // CELL * ncx * 4
    vx, vy = dirs[:, 0].astype(F), dirs[:, 1].astype(F)
    with np.errstate(all="ignore"):
        n1 = np.sqrt((vx.astype(np.float64) * vx + (vy * vy).astype(np.float64)).astype(F))
    ok = (n1 > F(1e-6)) & (n1 < np.inf)
    c = xy[ok].astype(F)
    x, y = c[:, 0].astype(np.int64), c[:, 1].astype(np.int64)
    sub = ((y // CELL) * ncx + x // CELL) * 4 + (y % CELL) // SUB * 2 + (x % CELL) // SUB
    bins = np.minimum(NBIN - 1, (pseudo_angle(vx[ok], vy[ok]) * F(NBIN // 4)).astype(np.int64))
    hist = np.zeros((nsub, NBIN), np.int64)
    np.add.at(hist, (sub, bins), 1)
    box = np.tile(np.array([np.inf, -np.inf, np.inf, -np.inf], F), (nsub, 1))
    np.minimum.at(box[:, 0], sub, c[:, 0])
    np.maximum.at(box[:, 1], sub, c[:, 0])
    np.minimum.at(box[:, 2], sub, c[:, 1])
    np.maximum.at(box[:, 3], sub, c[:, 1])
    rec = np.empty((nsub, REC), np.int32)
    rec[:, :4] = box.view(np.int32)
    rec[:, 4:] = np.cumsum(hist, 1).astype("<u2").view(np.int32)
    return rec.reshape(nsub // 4, 4, REC)


def pass_lists(bnd, b2, cnt):
    """The two lists the kernels score, each in index order: pass 1 = the PASS1 largest bounds B (prune_bound_kernel),
    pass 2 = every other h with B(h) >= L and B2(h) >= L (prune_next_kernel), L the best exact count of pass 1;
    b2 = count_bound over the sub-cell records.  Also the pass-2 list without the sub-cell refinement."""
    p1 = np.sort(np.argsort(-bnd, kind="stable")[:PASS1])
    rest = np.ones(len(bnd), bool)
    rest[p1] = False
    L = cnt[p1].max() if len(p1) else 0
    coarse = rest & (bnd >= L)
    return p1, np.nonzero(coarse & (b2 >= L))[0], np.nonzero(coarse)[0]
