"""CPU tests of the oracle (oracle/pvnet_oracle.c): known-answer and analytic checks.
The reference ships no tests for this path (SURVEY.md section 4); these pin the restatement's
semantics, tests/test_golden.py pins it against outputs of the reference extension itself."""
import math

import numpy as np
import pytest


def test_philox_known_answers(oracle):
    # Random123 kat_vectors, philox4x32-10
    kats = [
        ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
        ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
        ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
         [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
    ]
    for ctr, key, exp in kats:
        assert [int(x) for x in oracle.philox4x32_10(ctr, key)] == exp


def _field(kp, coords, noise=None):
    d = kp[None, :, :] - coords[:, None, :]
    d = d / np.linalg.norm(d, axis=2, keepdims=True)
    return d.astype(np.float32)


def test_hypothesis_is_ray_intersection(oracle):
    rng = np.random.default_rng(0)
    coords = rng.integers(0, 200, size=(50, 2)).astype(np.float32)
    kp = np.array([[77.25, 31.5], [300.0, -40.0]], dtype=np.float32)
    direct = _field(kp, coords)
    idxs = rng.integers(0, 50, size=(64, 2, 2)).astype(np.int32)
    hyp = oracle.generate_hypothesis(direct, coords, idxs)
    for h in range(64):
        for k in range(2):
            t0, t1 = idxs[h, k]
            if t0 == t1:
                assert tuple(hyp[h, k]) == (0.0, 0.0)      # degenerate pair keeps the zero fill (.cu:42-43,75)
            elif abs(direct[t0, k, 0] * direct[t1, k, 1] - direct[t0, k, 1] * direct[t1, k, 0]) > 1e-3:
                assert np.allclose(hyp[h, k], kp[k], atol=2e-2)


def test_parallel_rays_give_zero(oracle):
    coords = np.array([[0, 0], [10, 0]], dtype=np.float32)
    direct = np.array([[[0, 1]], [[0, 1]]], dtype=np.float32)
    hyp = oracle.generate_hypothesis(direct, coords, np.array([[[0, 1]]], dtype=np.int32))
    assert tuple(hyp[0, 0]) == (0.0, 0.0)


def test_vote_predicate_edges(oracle):
    coords = np.array([[0, 0], [5, 5], [9, 0]], dtype=np.float32)
    direct = np.array([[[1, 0]], [[0, 0]], [[-1, 0]]], dtype=np.float32)   # pixel 1 has a zero vector
    hyp = np.array([[[20, 0]], [[5, 5]], [[0, 0]]], dtype=np.float32)
    inl = np.zeros((3, 1, 3), dtype=np.uint8)
    oracle.voting_for_hypothesis(direct, coords, hyp, inl, 0.99)
    # hyp (20,0): pixel 0 points at it, pixel 1 never votes, pixel 2 points away
    assert inl[0, 0].tolist() == [1, 0, 0]
    # hyp coincident with pixel 1: norm2 < 1e-6 there; others off-axis
    assert inl[1, 0].tolist() == [0, 0, 0]
    # hyp (0,0) coincides with pixel 0 (no vote); pixel 2 points straight at it
    assert inl[2, 0].tolist() == [0, 0, 1]
    # voting only sets bytes, never clears
    inl2 = np.full((3, 1, 3), 7, dtype=np.uint8)
    oracle.voting_for_hypothesis(direct, coords, hyp, inl2, 0.99)
    assert inl2[0, 0].tolist() == [1, 7, 7]
    assert (oracle.vote_count(direct, coords, hyp, 0.99)[:, 0] == inl.sum(axis=2)[:, 0]).all()


def test_threshold_is_strict_and_fp32(oracle):
    # cos exactly equal to the fp32 threshold must not vote (.cu:124 uses >)
    coords = np.array([[0, 0]], dtype=np.float32)
    direct = np.array([[[1, 0]]], dtype=np.float32)
    hyp = np.array([[[3, 0]]], dtype=np.float32)     # cos == 1.0 exactly
    assert oracle.vote_count(direct, coords, hyp, 1.0)[0, 0] == 0
    assert oracle.vote_count(direct, coords, hyp, float(np.nextafter(np.float32(1), np.float32(0))))[0, 0] == 1


def _make_image(H, W, K, kp, fill_rect, seed=0, outliers=0.0, zero_bg=False):
    rng = np.random.default_rng(seed)
    mask = np.zeros((H, W), dtype=np.int64)
    y0, y1, x0, x1 = fill_rect
    mask[y0:y1, x0:x1] = 1
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    v = np.stack([kp[None, None, :, 0] - xx[:, :, None], kp[None, None, :, 1] - yy[:, :, None]], axis=-1)
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    v = v / np.maximum(n, 1e-12)
    if outliers:
        ang = rng.uniform(0, 2 * np.pi, size=(H, W, K))
        rv = np.stack([np.cos(ang), np.sin(ang)], axis=-1)
        sel = rng.uniform(size=(H, W, K)) < outliers
        v = np.where(sel[..., None], rv, v)
    bg = rng.uniform(0, 2 * np.pi, size=(H, W, K))
    bgv = np.stack([np.cos(bg), np.sin(bg)], axis=-1) * (0.0 if zero_bg else 1.0)
    v = np.where(mask[:, :, None, None] == 1, v, bgv)
    return mask, v.astype(np.float32)


def test_v3_recovers_keypoints(oracle):
    H, W, K = 60, 80, 3
    kp = np.array([[20.3, 30.7], [70.1, 10.2], [130.0, 25.0]], dtype=np.float32)   # last one outside the image
    mask, vertex = _make_image(H, W, K, kp, (10, 50, 15, 65))
    out, dbg = oracle.ransac_voting_layer_v3(mask[None], vertex[None], 64, inlier_thresh=0.99, seed=7, debug=True)
    assert dbg["tn"][0] == 40 * 50
    assert np.abs(out[0] - kp).max() < 2e-3          # noise-free field: least squares recovers the keypoint
    # 30 % random directions: those inside the 8-degree cone bias the fit a little, RANSAC still locks on
    mask_o, vertex_o = _make_image(H, W, K, kp, (10, 50, 15, 65), outliers=0.3)
    out_o = oracle.ransac_voting_layer_v3(mask_o[None], vertex_o[None], 64, inlier_thresh=0.99, seed=7)
    assert np.abs(out_o[0] - kp).max() < 1.5
    # batch composition / img_base do not change an image's result
    out2 = oracle.ransac_voting_layer_v3(np.stack([mask * 0, mask]), np.stack([vertex, vertex]), 64,
                                         inlier_thresh=0.99, seed=7, img_base=-1)
    assert (out2[0] == 0).all()                       # fg < min_num -> zeros (:129-132)
    assert np.array_equal(out2[1], out[0])


def test_v3_thinning_and_selection(oracle):
    H, W, K = 64, 64, 2
    kp = np.array([[10.5, 50.25], [40.0, 8.0]], dtype=np.float32)
    mask, vertex = _make_image(H, W, K, kp, (0, 64, 0, 64))
    rng = np.random.default_rng(3)
    sel = rng.uniform(size=(1, H, W)).astype(np.float32)
    out, dbg = oracle.ransac_voting_layer_v3(mask[None], vertex[None], 32, inlier_thresh=0.99, max_num=500,
                                             selection=sel, seed=1, debug=True)
    ratio = np.float32(500) / np.float32(4096)
    assert dbg["tn"][0] == int((sel[0] < ratio).sum())
    assert np.abs(out[0] - kp).max() < 5e-2
    out_p, dbg_p = oracle.ransac_voting_layer_v3(mask[None], vertex[None], 32, inlier_thresh=0.99, max_num=500,
                                                 seed=11, debug=True)
    assert abs(int(dbg_p["tn"][0]) - 500) < 5 * math.sqrt(500)
    assert np.abs(out_p[0] - kp).max() < 5e-2


def test_v3_mask_byte_semantics(oracle):
    # cur_mask = mask.byte(): 256 wraps to 0, 2 is foreground and counts twice in foreground_num (:125-126)
    H, W, K = 16, 16, 1
    kp = np.array([[8.2, 3.1]], dtype=np.float32)
    mask, vertex = _make_image(H, W, K, kp, (0, 16, 0, 16))
    m = mask.copy()
    m[:, :8] = 256
    m[:, 8:] = 2
    out, dbg = oracle.ransac_voting_layer_v3(m[None], vertex[None], 16, inlier_thresh=0.99, max_num=200,
                                             selection=np.zeros((1, H, W), np.float32), debug=True)
    # fg = 2*128 = 256 > max_num -> thinning active, selection 0 keeps everything that is non-zero
    assert dbg["tn"][0] == 128


def test_distribution_matches_numpy(oracle):
    H, W, K = 40, 48, 2
    kp = np.array([[20.0, 20.0], [60.0, 5.0]], dtype=np.float32)
    mask, vertex = _make_image(H, W, K, kp, (5, 35, 5, 40), outliers=0.2, seed=5)
    mean = kp[None].copy()
    _, cov, dbg = oracle.estimate_voting_distribution_with_mean(mask[None], vertex[None], mean, round_hyp_num=32,
                                                                min_hyp_num=128, seed=9, debug=True)
    hyp, ratio = dbg["hyp"][0], dbg["ratio"][0]      # [K,hn,2], [K,hn]
    for k in range(K):
        w = ratio[k].astype(np.float64).copy()
        w[ratio[k] < ratio[k].max() - np.float32(0.1)] = 0
        d = (hyp[k] - mean[0, k]).astype(np.float64)
        ref = (d.T * w) @ d / (np.float32(w.sum()) + np.float32(1e-3))
        assert np.allclose(cov[0, k], ref, rtol=1e-5, atol=1e-6)
    # fewer than min_num pixels: hyp zeros, ratio ones (:211-216)
    _, cov0 = oracle.estimate_voting_distribution_with_mean(mask[None] * 0, vertex[None], mean, 32, 128)
    exp = np.einsum("ki,kj->kij", mean[0], mean[0]) * 128 / (np.float32(128) + np.float32(1e-3))
    assert np.allclose(cov0[0], exp, rtol=1e-5)


def test_vanishing_point_pair(oracle):
    rng = np.random.default_rng(2)
    coords = rng.integers(0, 100, size=(40, 2)).astype(np.float32)
    kp = np.array([[150.5, 60.25]], dtype=np.float32)
    direct = _field(kp, coords)
    idxs = rng.integers(0, 40, size=(32, 1, 2)).astype(np.int32)
    hyp = oracle.generate_hypothesis(direct, coords, idxs, vanishing_point=True)
    ok = 0
    for h in range(32):
        x, y, z = hyp[h, 0]
        if abs(z) > 1e-3:
            assert np.allclose([x / z, y / z], kp[0], atol=5e-2)
            ok += 1
    assert ok > 10
    inl = np.zeros((32, 1, 40), dtype=np.uint8)
    oracle.voting_for_hypothesis(direct, coords, hyp, inl, 0.999, vanishing_point=True)
    good = [h for h in range(32) if abs(hyp[h, 0, 2]) > 1e-3]
    assert inl[good].mean() > 0.9


def test_cfg1_cpu_plumbing_case(oracle):
    """BASELINE.json configs[0] ("single 128x128 synthetic mask + random unit-vector field, K=1, 64 hypotheses, CPU
    reference path, plumbing, no GPU"): the oracle end to end on the CPU.  A pure random field has no consensus, so the
    checks are structural: determinism, the winner is the first maximum of the counts, the counts equal the byte-tensor
    formulation (voting_for_hypothesis + sum, ransac_voting_gpu.py:156-159), the refit is the least-squares point of the
    winner's inliers, and the distribution op runs.  tests/test_gpu_configs.py::test_cfg1_plumbing_case compares the CUDA
    path with exactly this."""
    import time
    import torch
    from clean_pvnet_b200 import synth
    mask, vertex, _ = synth.make_inputs("cfg1", device="cpu", seed=1235)
    m, v = mask.numpy(), vertex.numpy()
    assert m.shape == (1, 128, 128) and v.shape == (1, 128, 128, 1, 2)
    t0 = time.perf_counter()
    out, dbg = oracle.ransac_voting_layer_v3(m, v, 64, inlier_thresh=0.99, seed=11, debug=True)
    dt = time.perf_counter() - t0
    out2 = oracle.ransac_voting_layer_v3(m, v, 64, inlier_thresh=0.99, seed=11)
    assert np.array_equal(out, out2) and np.isfinite(out).all()
    tn = int(dbg["tn"][0])
    assert tn == int(m.sum()) and 4000 < tn < 6000                    # ~30 % of 128*128, below max_num: no thinning
    yx = np.argwhere(m[0] != 0)                                        # row-major = torch.nonzero order (:140)
    coords = np.ascontiguousarray(yx[:, ::-1].astype(np.float32))      # (x, y)                      (:141)
    direct = np.ascontiguousarray(v[0][m[0] != 0])                     # [tn,1,2] masked_select      (:142-143)
    hyp = np.ascontiguousarray(dbg["hyp"][0].transpose(1, 0, 2))       # [hn,1,2]
    inl = np.zeros((64, 1, tn), np.uint8)
    oracle.voting_for_hypothesis(direct, coords, hyp, inl, 0.99)
    counts = inl.sum(2).T                                              # [1,64]
    assert np.array_equal(counts, dbg["counts"][0])
    h = int(np.argmax(counts[0]))                                      # first maximum, like torch.max
    assert np.array_equal(dbg["win"][0, 0], hyp[h, 0])
    w = inl[h, 0].astype(np.float64)
    n = np.stack([direct[:, 0, 1], -direct[:, 0, 0]], 1).astype(np.float64) * w[:, None]
    b = (n * coords).sum(1)
    x = np.linalg.solve(n.T @ n, n.T @ b)
    assert np.abs(x - out[0, 0]).max() < 1e-3
    _, cov = oracle.estimate_voting_distribution_with_mean(m, v, out, seed=12)
    assert cov.shape == (1, 1, 2, 2) and np.isfinite(cov).all()
    assert dt < 5.0                                                    # 64 x 5 000 tests: milliseconds on one core


def _torch_select(mask, mode, min_num, max_num, selection):
    """The reference's selection ops, one image at a time on CPU tensors (ransac_voting_gpu.py:125-143 for mode 0,
    :205-227 for mode 1): fg, nz, tn (-1 = skipped) and the row-major indices torch.nonzero returns."""
    import torch
    res = []
    for bi in range(mask.shape[0]):
        cur_mask = mask[bi].byte() if mode == 0 else (mask[bi] == 1)
        foreground_num = torch.sum(cur_mask)
        nz = int(torch.count_nonzero(cur_mask))
        if foreground_num < min_num:
            res.append((int(foreground_num), nz, -1, np.zeros(0, np.int64)))
            continue
        if foreground_num > max_num:
            selected_mask = selection[bi] < (max_num / foreground_num.float())   # fp32, strict
            cur_mask = cur_mask * selected_mask.to(cur_mask.dtype)
        pix = torch.nonzero(cur_mask.reshape(-1))[:, 0].numpy()
        res.append((int(foreground_num), nz, len(pix), pix))
    return res


def test_select_pixels_matches_torch_ops(oracle):
    """orc_select_pixels with explicit draws against the reference's own torch ops: byte values (wrap-around, sums of
    values above 1), `== 1` for the distribution op, the fp32 ratio `max_num / fg.float()` (torch evaluates it as
    reciprocal() * max_num) compared strictly, draws placed exactly on that ratio, one ulp below it and at 0."""
    import torch
    rng = np.random.default_rng(21)
    B, H, W = 12, 37, 53
    vals = np.array([0, 0, 0, 0, 1, 1, 1, 2, 3, 255, 256, 257, -1, -255, 2 ** 32 + 1], np.int64)
    mask = np.zeros((B, H, W), np.int64)
    for b in range(B):
        fill = [0.02, 0.1, 0.3, 0.6, 0.9][b % 5]
        on = rng.uniform(size=(H, W)) < fill
        mask[b] = np.where(on, rng.choice(vals, size=(H, W)), 0)
    mask[11] = 0
    mask[11, 3, 2:6] = 1                                   # 4 pixels: skipped at min_num 5 (both modes)
    sel = rng.uniform(size=(B, H, W)).astype(np.float32)
    mt, st = torch.from_numpy(mask), torch.from_numpy(sel)
    for mode in (0, 1):
        for max_num in (40, 200, 30000):
            # plant draws on the ratio boundary of every thinned image
            fgs = [r[0] for r in _torch_select(mt, mode, 5, max_num, st)]
            s2 = sel.copy()
            for b, fg in enumerate(fgs):
                if fg > max_num:
                    ratio = (torch.tensor(fg).float().reciprocal() * max_num).item()
                    r32 = np.float32(ratio)
                    assert r32 == (max_num / torch.tensor(fg).float()).item()
                    on = np.flatnonzero(mask[b].reshape(-1) != 0)
                    s2[b].reshape(-1)[on[0::3]] = r32                                        # dropped
                    s2[b].reshape(-1)[on[1::3]] = np.nextafter(r32, np.float32(0))           # kept
                    s2[b].reshape(-1)[on[2::7]] = 0.0                                        # kept
            want = _torch_select(mt, mode, 5, max_num, torch.from_numpy(s2))
            got = oracle.select_pixels(mask, mode, 5, max_num, selection=s2)
            for b in range(B):
                fg, nz, tn, pix = want[b]
                assert (int(got["fg"][b]), int(got["nz"][b]), int(got["tn"][b])) == (fg, nz, tn), (mode, max_num, b)
                assert np.array_equal(got["pix"][b], pix), (mode, max_num, b)
    # the value semantics the expectations above rest on
    assert mt.byte()[mt == 256].eq(0).all() and mt.byte()[mt == -1].eq(255).all() and mt.byte()[mt == 2 ** 32 + 1].eq(1).all()
    # the ratio is NOT the correctly rounded quotient for every fg: the oracle must follow torch where they differ
    fg = 30001
    assert np.float32(30000) / np.float32(fg) != (30000 / torch.tensor(fg).float()).item()
    m1 = np.ones((1, 1, fg), np.int64)
    r = np.float32((30000 / torch.tensor(fg).float()).item())
    s1 = np.full((1, 1, fg), 0.99999, np.float32)
    s1[0, 0, :5] = [r, np.nextafter(r, np.float32(2)), np.nextafter(r, np.float32(0)), 0.0, np.float32(30000) / np.float32(fg)]
    got = oracle.select_pixels(m1, 0, 5, 30000, selection=s1)
    assert got["tn"][0] == 2 + (s1[0, 0, 4] < r) and list(got["pix"][0][:2]) == [2, 3]
    # philox draws (selection=None) follow the tag: v3 and the distribution op thin with different streams
    a = oracle.select_pixels(mask, 0, 5, 40, seed=5)
    b = oracle.select_pixels(mask, 0, 5, 40, seed=5, tag=4)
    assert np.array_equal(a["fg"], b["fg"]) and any(not np.array_equal(x, y) for x, y in zip(a["pix"], b["pix"]))
