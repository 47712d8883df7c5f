"""GPU: the pruned v3 vote's list kernel (vote_list_kernel, csrc/vote.cu) on inputs that reach its guard band, its exact path
and every chunk of pass 2.

Bars: keypoints bit-identical to the same call with every hypothesis scored (debug=True); every hypothesis the two passes
scored has debug=True's count, every other one count 0.  Pruning runs on every input here (t = 0.99, hn = 512,
B*K = 36 >= 32)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HN, THRESH, B, K, H, W = 512, 0.99, 4, 9, 480, 640


def _check(pvb, mask, vertex, seed, idxs=None):
    """pruned == full; returns the pass lists [2][B][K][hn] and lengths [2][B][K] of the pruned call"""
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    out = pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=seed, idxs=idxs)
    torch.cuda.synchronize()
    lib = _lib.load()
    m, v = rv._check_inputs(mask, vertex)
    d = rv._make_desc(m, v, HN, THRESH, 5, 30000, _lib.PVB_SELECT_BYTE, seed, 0, None)
    ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
    L = _lib.PvbLayout()
    _lib.check(lib.pvb_workspace_layout(d, L))
    lists = ws[L.prune_list:L.prune_list + 2 * B * K * HN * 4].view(torch.int32).view(2, B, K, HN).cpu().numpy()
    lens = ws[L.prune_len:L.prune_len + 2 * B * K * 4].view(torch.int32).view(2, B, K).cpu().numpy()
    cp = rv._views(ws, d, lib)["counts"].cpu().numpy()
    full, dbg = pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=seed, idxs=idxs, debug=True)
    assert torch.equal(out.view(torch.int32), full.view(torch.int32)), "keypoints differ from the full path"
    cf = dbg["counts"].cpu().numpy()
    for b in range(B):
        for k in range(K):
            scored = np.zeros(HN, bool)
            for p in range(2):
                scored[lists[p, b, k, :lens[p, b, k]]] = True
            assert lens[0, b, k] + lens[1, b, k] == scored.sum(), "a hypothesis was listed twice"
            assert np.array_equal(cp[b, k][scored], cf[b, k][scored]), f"image {b} keypoint {k}: counts differ"
            assert (cp[b, k][~scored] == 0).all()
    return lists, lens


def test_list_kernel_guard_band_on_ray_intersections(pvb):
    """Noise-free rays toward keypoints on exact pixel centres; every hypothesis intersects two of them, so it lies within
    a few ulps of the keypoint.  The bounds tie, pass 1 takes 128 hypotheses by index and pass 2 the rest, and the pixel
    at the keypoint sits inside the guard band of every hypothesis: the exact path decides it in both passes."""
    rng = np.random.default_rng(5)
    yy, xx = np.mgrid[0:H, 0:W]
    cx, cy, r = 320, 240, 60
    disc = (xx - cx) ** 2 + (yy - cy) ** 2 <= r * r                      # ~11 300 pixels: below max_num, no thinning
    ys, xs = np.nonzero(disc)                                           # the selected pixels, in torch.nonzero order
    mask = np.broadcast_to(disc, (B, H, W)).astype(np.int64)
    vertex = np.zeros((B, H, W, K, 2), np.float32)
    idxs = np.zeros((B, HN, K, 2), np.int32)
    for b in range(B):
        for k in range(K):
            kx, ky = cx - 24 + 6 * k + b, cy - 12 + 3 * k - 2 * b       # integer: an exact pixel centre inside the disc
            dx, dy = kx - xx.astype(np.float64), ky - yy.astype(np.float64)
            n = np.hypot(dx, dy)
            n[ky, kx] = 1.0
            vx, vy = dx / n, dy / n
            vx[ky, kx], vy[ky, kx] = 1.0, 0.0                           # the pixel at the keypoint: any direction
            vertex[b, :, :, k, 0], vertex[b, :, :, k, 1] = vx, vy
            # pairs of pixels whose rays cross at 0.5..2.6 rad: well-conditioned intersections
            ang = np.arctan2(ky - ys, kx - xs)
            ok = ~((xs == kx) & (ys == ky))
            pairs = []
            while len(pairs) < HN:
                i, j = rng.integers(0, len(xs), 2)
                d = abs((ang[i] - ang[j] + math.pi) % (2 * math.pi) - math.pi)
                if ok[i] and ok[j] and 0.5 < d < 2.6:
                    pairs.append((i, j))
            idxs[b, :, k] = pairs
    mask_t, vertex_t = torch.from_numpy(mask).cuda(), torch.from_numpy(vertex).cuda()
    idxs_t = torch.from_numpy(idxs).cuda()
    _, dbg = pvb.ransac_voting_layer_v3(mask_t, vertex_t, HN, inlier_thresh=THRESH, seed=3, idxs=idxs_t, debug=True)
    hyp = dbg["hyp"].cpu().numpy().astype(np.float64)
    for b in range(B):
        for k in range(K):
            kp = np.array([cx - 24 + 6 * k + b, cy - 12 + 3 * k - 2 * b], np.float64)
            assert np.abs(hyp[b, k] - kp).max() < 1e-3                  # every hypothesis is (nearly) the keypoint
    _, lens = _check(pvb, mask_t, vertex_t, 3, idxs=idxs_t)
    assert (lens[0] == 128).all()
    assert (lens[1] >= 300).all(), lens[1]


def test_list_kernel_guard_band_on_distinct_hypotheses(pvb):
    """Random directions, except that hypothesis j is the crossing of two rays aimed at its own pixel r_j: 512 distinct
    hypotheses per (image, keypoint), each within ulps of a different pixel, which is inside its guard band.  The exact
    path must re-test r_j against hypothesis j itself, not against another entry of the list."""
    rng = np.random.default_rng(7)
    yy, xx = np.mgrid[0:H, 0:W]
    cx, cy, r = 320, 240, 60
    disc = (xx - cx) ** 2 + (yy - cy) ** 2 <= r * r                      # ~11 300 pixels: below max_num, no thinning
    ys, xs = np.nonzero(disc)
    mask = np.broadcast_to(disc, (B, H, W)).astype(np.int64)
    ang = rng.uniform(0, 2 * math.pi, (B, H, W, K))
    vertex = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)
    idxs = np.zeros((B, HN, K, 2), np.int32)
    target = np.zeros((B, K, HN, 2))
    for b in range(B):
        for k in range(K):
            perm = iter(rng.permutation(len(xs)))
            for j in range(HN):
                t = next(perm)
                while True:
                    p, q = next(perm), next(perm)
                    a_p = math.atan2(ys[t] - ys[p], xs[t] - xs[p])
                    a_q = math.atan2(ys[t] - ys[q], xs[t] - xs[q])
                    if 0.5 < abs((a_p - a_q + math.pi) % (2 * math.pi) - math.pi) < 2.6:
                        break
                for s in (p, q):
                    d = np.array([xs[t] - xs[s], ys[t] - ys[s]], np.float64)
                    vertex[b, ys[s], xs[s], k] = d / np.hypot(*d)
                idxs[b, j, k] = (p, q)
                target[b, k, j] = (xs[t], ys[t])
    mask_t, vertex_t = torch.from_numpy(mask).cuda(), torch.from_numpy(vertex).cuda()
    idxs_t = torch.from_numpy(idxs).cuda()
    _, dbg = pvb.ransac_voting_layer_v3(mask_t, vertex_t, HN, inlier_thresh=THRESH, seed=5, idxs=idxs_t, debug=True)
    hyp = dbg["hyp"].cpu().numpy().astype(np.float64)
    assert np.abs(hyp - target).max() < 1e-3                            # hypothesis j sits on its pixel r_j
    _, lens = _check(pvb, mask_t, vertex_t, 5, idxs=idxs_t)
    assert (lens[1] >= 300).all(), lens[1]


def test_list_kernel_bad_vectors(pvb):
    """Zero, NaN, +-inf and 1e30 vectors in a cfg-2 field: pixels that never vote, pixels forced onto the exact path, and
    non-finite or huge hypotheses, which every pixel re-tests exactly (padding must stay out of it)."""
    from clean_pvnet_b200 import synth
    mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=81, B=B)
    vertex = vertex.clone()
    g = torch.Generator(device="cuda").manual_seed(82)
    fg = mask.nonzero()
    bad = [(0.0, 0.0), (float("nan"), 1.0), (float("inf"), 0.0), (0.0, -float("inf")), (1e30, -1e30)]
    for i, val in enumerate(bad):
        pick = fg[torch.randint(0, fg.shape[0], (3000,), generator=g, device="cuda")]
        k = i % K
        vertex[pick[:, 0], pick[:, 1], pick[:, 2], k] = torch.tensor(val, device="cuda")
        vertex[pick[:, 0], pick[:, 1], pick[:, 2], (k + 4) % K] = torch.tensor(val, device="cuda")
    _check(pvb, mask, vertex, 83)


def test_list_kernel_random_field_fills_every_chunk(pvb):
    """Uniformly random directions: the bound excludes (almost) nothing, so pass 2 fills all six chunks of 64 entries"""
    from clean_pvnet_b200 import synth
    cfg = dict(synth.CONFIGS["cfg2"], random_field=True)
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=91, B=B)
    _, lens = _check(pvb, mask, vertex, 92)
    assert (lens[1] > 64 * 5).all(), lens[1]                            # every pass-2 chunk 0..5 is non-empty
