"""The cell records and 128-bin bound of the pruned v3 vote (csrc/prune.cu, DESIGN.md 4.2).

The bound is summed over the 32x32-pixel cells of the image.  A numpy twin of prune_hist_kernel + count_bound (float32 like
the kernels) must give B(h) >= the oracle's count for every hypothesis: the pruned vote skips exactly the hypotheses whose
bound is below an exact count, so a bound below a count could change the winner.  On the CPU: production shapes at four
thresholds, and inputs built on the cell borders.  On the GPU: the kernel's cell records equal the twin's bit for bit, and
the two passes score at most 0.45 of the hypotheses on cfg-2."""
import math

import numpy as np
import pytest

import pvnet_oracle as po
from clean_pvnet_b200 import synth
from test_prune_bound import prune_rotation, pseudo_angle

CELL, NBIN = 32, 128             # PRUNE_CELL, PRUNE_NBIN (csrc/kernels.h)
REC = 4 + NBIN // 2              # PRUNE_REC: box (4 floats), then 16-bit inclusive prefix counts
EPS = np.float32(1e-5)
PASS1 = 128                      # PRUNE_M
F = np.float32


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
    """Slots the two passes fill: the PASS1 largest bounds (ties in index order), then every other h with B(h) >= L,
    L the best exact count of pass 1"""
    p1 = np.argsort(-bnd, kind="stable")[:PASS1]
    rest = np.ones(len(bnd), bool)
    rest[p1] = False
    return PASS1 + int(np.count_nonzero(rest & (bnd >= cnt[p1].max())))


def _check(xy, dirs, hyp, t, H, W):
    cnt = po.vote_count(dirs[:, None, :], xy, hyp[:, None, :], t)[:, 0]
    bnd = count_bound(hyp, cell_records(xy, dirs, H, W), len(xy), prune_rotation(t))
    bad = np.nonzero(bnd < cnt)[0]
    assert bad.size == 0, f"bound below count at t={t}: h={hyp[bad[:3]]} bound={bnd[bad[:3]]} count={cnt[bad[:3]]}"


def _layer_case(cfg, B, t, seed):
    """B(h) >= count(h) for every (image, keypoint, hypothesis); returns the scored fraction per (image, keypoint)"""
    mask, vertex, _ = synth.make_inputs(cfg, device="cpu", seed=seed, B=B)
    m, v = mask.numpy(), vertex.numpy()
    hn = synth.CONFIGS[cfg]["hn"]
    _, dbg = po.ransac_voting_layer_v3(m, v, hn, inlier_thresh=t, seed=seed, debug=True)
    sel = po.select_pixels(m, mode=0, seed=seed)
    H, W = m.shape[1:]
    frac = []
    for b in range(B):
        pix = sel["pix"][b]
        if len(pix) == 0:
            continue
        xy = np.stack([pix % W, pix // W], 1).astype(F)
        for k in range(v.shape[3]):
            rec = cell_records(xy, v[b, pix // W, pix % W, k].astype(F), H, W)
            bnd = count_bound(dbg["hyp"][b, k].astype(F), rec, len(pix), prune_rotation(t))
            cnt = dbg["counts"][b, k]
            assert np.all(bnd >= cnt), (cfg, b, k, t)
            frac.append(scored(bnd, cnt) / hn)
    return np.array(frac)


@pytest.mark.parametrize("cfg", ["cfg2", "cfg3", "cfg4", "cfg5"])
@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_cell_bound_production_shapes(cfg, t):
    _layer_case(cfg, 1, t, 1236)


def test_cell_bound_scores_under_045_on_cfg2():
    frac = _layer_case("cfg2", 2, 0.99, 1236)
    assert frac.mean() <= 0.45, frac.mean()


def _field(xy, kp, rng, noise=0.02):
    d = kp[None, :] - xy
    a = np.arctan2(d[:, 1], d[:, 0]) + rng.normal(0, noise, len(xy))
    return np.stack([np.cos(a), np.sin(a)], 1).astype(F)


@pytest.mark.parametrize("t", [0.5, 0.9, 0.99, 0.999])
def test_cell_bound_adversarial(t):
    """A 75 x 101 image (neither side a multiple of 32): a block straddling the cell borders x = 31/32, 63/64 and
    y = 31/32, single-pixel cells, cells whose every vector is zero, NaN or below the norm cut, and hypotheses inside the
    boxes, within half a pixel of them and on the cell corners."""
    rng = np.random.default_rng(15)
    H, W = 75, 101
    ys, xs = np.mgrid[24:40, 26:70]
    pts = [np.stack([xs.ravel(), ys.ravel()], 1)]
    pts.append(np.array([[5, 5], [100, 3], [3, 74], [100, 74], [31, 70], [32, 70], [96, 64]]))   # single-pixel cells
    pts.append(np.stack(np.meshgrid(np.arange(66, 70), np.arange(66, 70)), -1).reshape(-1, 2))  # all-zero cell
    pts.append(np.stack(np.meshgrid(np.arange(70, 74), np.arange(45, 48)), -1).reshape(-1, 2))  # all-NaN cell
    pts.append(np.stack(np.meshgrid(np.arange(10, 14), np.arange(40, 44)), -1).reshape(-1, 2))  # below the norm cut
    xy = np.concatenate(pts).astype(F)
    order = np.lexsort((xy[:, 0], xy[:, 1]))             # raster order, as the selected-pixel list
    groups = np.concatenate([np.full(len(p), i) for i, p in enumerate(pts)])[order]
    xy = xy[order]
    hyp = [[26, 24], [69, 39], [31, 31], [32, 32], [31.5, 31.5], [32, 31], [31, 32], [63.5, 31.5], [64, 32],
           [25.5, 24], [25.49, 24], [69.51, 39.49], [45, 23.5], [45, 23.49], [45, 40.49], [5, 5], [5.5, 5.5], [5.51, 5],
           [96, 96], [0, 0], [32, 0], [0, 32], [64, 64], [96, 32], [100.5, 74.5], [50, 200], [-40, 30], [1e6, 3],
           [np.nan, 4], [np.inf, 1], [1e16, 0]]
    hyp = np.concatenate([np.array(hyp, F), rng.uniform(-20, 120, (60, 2)).astype(F)])
    for aim in ([31.5, 31.5], [25.49, 24], [64, 32], [5.51, 5], [50, 200]):
        dirs = _field(xy, np.array(aim), rng, noise=0.0 if aim[0] == 64 else 0.01)
        dirs[groups == 2] = 0.0
        dirs[groups == 3] = np.nan
        dirs[groups == 4] *= F(1e-7)
        _check(xy, dirs, hyp, t, H, W)
        rec = cell_records(xy, dirs, H, W)
        tot = rec[:, -1].astype(np.int64) >> 16
        assert tot.sum() == np.count_nonzero(groups < 2)  # the zero, NaN and tiny vectors are in no cell


@pytest.mark.gpu
def test_gpu_cell_records_and_scored_fraction(pvb):
    """The kernel's cell records (read from the workspace like tests/test_gpu_prune.py reads the lists) equal the twin's
    bit for bit, and the mean pass-1 + pass-2 length on cfg-2 is at most 0.45 hn."""
    import torch
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=1236, B=4)
    hn, t = 512, 0.99
    pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=t, seed=1000)
    torch.cuda.synchronize()
    lib = _lib.load()
    m, v = rv._check_inputs(mask, vertex)
    d = rv._make_desc(m, v, hn, t, 5, 30000, _lib.PVB_SELECT_BYTE, 1000, 0, None)
    ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
    views = rv._views(ws, d, lib, refit=True)
    L = _lib.PvbLayout()
    _lib.check(lib.pvb_workspace_layout(d, L))
    B, K, H, W = d.B, d.K, d.H, d.W
    assert L.prune_ncells == math.ceil(H / CELL) * math.ceil(W / CELL)
    cells = ws[L.prune_cells:L.prune_cells + B * K * L.prune_ncells * REC * 4].view(torch.int32)
    cells = cells.view(B, K, L.prune_ncells, REC).cpu().numpy()
    lens = ws[L.prune_len:L.prune_len + 2 * B * K * 4].view(torch.int32).view(2, B, K).cpu().numpy()
    tn = views["tn"].cpu().numpy()
    xy, dirs = views["xy"].cpu().numpy(), views["dirs"].cpu().numpy()
    for b in range(B):
        for k in range(K):
            want = cell_records(xy[b, :tn[b]], dirs[b, k, :tn[b]], H, W)
            bad = np.nonzero((cells[b, k] != want).any(1))[0]
            assert bad.size == 0, f"image {b} keypoint {k}: cells {bad[:4]} differ from the twin"
    frac = (lens[0] + lens[1]).mean() / hn
    print(f"cfg2 mean pass-1 + pass-2 length: {frac:.3f} hn")
    assert frac <= 0.45
