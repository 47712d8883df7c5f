"""GPU parity, operator level: ransac_voting_layer_v3 / estimate_voting_distribution_with_mean
through the C ABI against the CPU oracle on the same seeded inputs.

Bars: selected pixel lists, sample indices, hypotheses (bit pattern), inlier counts and winners are
exact; the refit's normal equations equal the sums over the reference predicate's inliers of the winner within rtol 1e-12
(summation order; one pixel more or less is far outside it); refit keypoints within 1e-4 px of the oracle (both accumulate in double; the reference's own
fp32 accumulation noise is ~1e-4 px, the north-star tolerance vs the reference is 1e-3 px);
covariances within 1 fp32 ulp of a float64 restatement of the covariance kernel (tests/util.py)."""
import numpy as np
import pytest
import torch

from util import bits_equal, check_covariance, check_normal_eq, oracle_inliers, twin_inliers

pytestmark = pytest.mark.gpu

KPT_TOL = 1e-4


def _inputs(pvb, cfg, seed=1234, **kw):
    from clean_pvnet_b200 import synth
    return synth.make_inputs(cfg, device="cuda", seed=seed, **kw)


def _np(*ts):
    return [t.detach().cpu().contiguous().numpy() for t in ts]


def _check_v3(pvb, oracle, mask, vertex, hn, thresh=0.99, seed=99, img_base=0, **kw):
    out, dbg = pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=thresh, seed=seed, img_base=img_base,
                                          debug=True, **kw)
    m, v = _np(mask, vertex)
    okw = {k: (_np(kw[k])[0] if kw.get(k) is not None else None) for k in ("idxs", "selection")}
    want, odbg = oracle.ransac_voting_layer_v3(m.astype(np.int64) if m.dtype != np.bool_ else m.astype(np.int64), v, hn,
                                               inlier_thresh=thresh, seed=seed, img_base=img_base, debug=True,
                                               min_num=kw.get("min_num", 5), max_num=kw.get("max_num", 30000), **okw)
    tn = dbg["tn"].cpu().numpy()
    assert np.array_equal(tn, odbg["tn"])
    assert bits_equal(dbg["hyp"].cpu().numpy(), odbg["hyp"])
    assert np.array_equal(dbg["counts"].cpu().numpy(), odbg["counts"])
    assert bits_equal(dbg["win"].cpu().numpy(), odbg["win"])
    check_normal_eq(dbg, thresh, oracle_inliers(oracle))
    got = out.cpu().numpy()
    assert np.isfinite(got).all()
    assert np.abs(got - want).max() < KPT_TOL
    return got, dbg, odbg


def test_v3_small_matches_oracle(pvb, oracle):
    mask, vertex, kp = _inputs(pvb, "small")
    got, dbg, _ = _check_v3(pvb, oracle, mask, vertex, 64)
    assert np.abs(got - kp.cpu().numpy())[:, :-1].max() < 8.0      # 3 deg noise + 20 % outliers on a 96x128 image: a few px


def test_v3_selection_order_and_gather(pvb):
    """xy[] is torch.nonzero order (row-major) and dirs[] holds vertex at those pixels."""
    mask, vertex, _ = _inputs(pvb, "small", seed=5)
    _, dbg = pvb.ransac_voting_layer_v3(mask, vertex, 16, inlier_thresh=0.99, debug=True)
    for b in range(mask.shape[0]):
        nzc = torch.nonzero(mask[b])[:, [1, 0]].float()
        tn = int(dbg["tn"][b])
        assert tn == nzc.shape[0]
        assert torch.equal(dbg["xy"][b, :tn], nzc)
        sel = vertex[b][mask[b] != 0]                                # [tn,K,2]
        assert torch.equal(dbg["dirs"][b, :, :tn].permute(1, 0, 2), sel)


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8, torch.bool, torch.int16, torch.int8,
                                   torch.float32, torch.float64])
def test_v3_mask_dtypes(pvb, oracle, dtype):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=3)
    ref = pvb.ransac_voting_layer_v3(mask, vertex, 32, inlier_thresh=0.99, seed=5)
    got = pvb.ransac_voting_layer_v3(mask.to(dtype), vertex, 32, inlier_thresh=0.99, seed=5)
    assert torch.equal(ref, got)


def test_v3_byte_wraparound_and_weights(pvb, oracle):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=4)
    m = mask.clone()
    m[mask == 1] = 2          # foreground value 2: still foreground, fg sum doubles
    m[:, :4, :] = 256         # wraps to 0 under .byte()
    _check_v3(pvb, oracle, m, vertex, 32, max_num=400)


def test_v3_strided_inputs(pvb, oracle):
    """The production call passes a permuted view of NCHW (resnet18.py:66-68) and sliced masks."""
    mask, vertex, _ = _inputs(pvb, "small", seed=6, layout="planar")
    assert not vertex.is_contiguous()
    got, _, _ = _check_v3(pvb, oracle, mask, vertex, 64)
    big = torch.zeros(mask.shape[0], mask.shape[1] * 2, mask.shape[2] * 2, dtype=mask.dtype, device="cuda")
    big[:, ::2, ::2] = mask
    mv = big[:, ::2, ::2]
    assert not mv.is_contiguous()
    got2 = pvb.ransac_voting_layer_v3(mv, vertex.contiguous(), 64, inlier_thresh=0.99, seed=99)
    assert np.array_equal(got2.cpu().numpy(), got)


def test_v3_thinning_philox_and_explicit(pvb, oracle):
    mask, vertex, _ = _inputs(pvb, "small", seed=7)
    got, dbg, _ = _check_v3(pvb, oracle, mask, vertex, 64, max_num=600)
    tn = dbg["tn"].cpu().numpy()
    assert (np.abs(tn - 600) < 6 * np.sqrt(600)).all()
    B, H, W = mask.shape
    g = torch.Generator(device="cuda").manual_seed(3)
    selection = torch.rand((B, H, W), generator=g, device="cuda")
    idxs = torch.randint(0, 300, (B, 64, vertex.shape[3], 2), generator=g, device="cuda", dtype=torch.int32)
    _check_v3(pvb, oracle, mask, vertex, 64, max_num=600, idxs=idxs, selection=selection)


def test_v3_skips_small_foreground(pvb, oracle):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=8)
    mask[0] = 0
    mask[0, 3, 3:7] = 1          # 4 < min_num pixels -> zeros (:129-132)
    got, dbg, _ = _check_v3(pvb, oracle, mask, vertex, 32)
    assert (got[0] == 0).all() and int(dbg["state"][0]) == 1 and int(dbg["state"][1]) == 0
    out = pvb.ransac_voting_layer_v3(mask, vertex, 32, inlier_thresh=0.99, min_num=4, seed=1)
    assert (out[0] != 0).any()


def test_v3_sharding_invariance(pvb):
    """An image's result depends on (seed, global image index) only -- not on batch composition."""
    mask, vertex, _ = _inputs(pvb, "small", seed=9, B=4)
    full = pvb.ransac_voting_layer_v3(mask, vertex, 64, inlier_thresh=0.99, seed=42, max_num=500)
    lo = pvb.ransac_voting_layer_v3(mask[:2], vertex[:2], 64, inlier_thresh=0.99, seed=42, max_num=500)
    hi = pvb.ransac_voting_layer_v3(mask[2:], vertex[2:], 64, inlier_thresh=0.99, seed=42, max_num=500, img_base=2)
    assert torch.equal(full, torch.cat([lo, hi]))
    again = pvb.ransac_voting_layer_v3(mask, vertex, 64, inlier_thresh=0.99, seed=42, max_num=500)
    assert torch.equal(full, again)


@pytest.mark.parametrize("hn", [1, 31, 128, 129, 256, 300, 512, 513, 1500])
def test_v3_hypothesis_counts(pvb, oracle, hn):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=10)
    _check_v3(pvb, oracle, mask, vertex, hn)


@pytest.mark.parametrize("H,W,K", [(45, 61, 2), (33, 31, 1), (135, 180, 5), (7, 300, 3)])
def test_v3_odd_image_sizes(pvb, oracle, H, W, K):
    """H*W not a multiple of 32 (partial bitmap word), odd widths, single keypoint."""
    cfg = dict(B=2, H=H, W=W, K=K, hn=40, fill=(0.3, 0.4), kind="blob")
    mask, vertex, _ = _inputs(pvb, cfg, seed=H * 1000 + W)
    _check_v3(pvb, oracle, mask, vertex, 40, max_num=200)
    _check_v3(pvb, oracle, mask, vertex, 40)


@pytest.mark.parametrize("case", range(24))
def test_v3_randomized_differential(pvb, oracle, case):
    """Random shapes / keypoint counts / hypothesis counts / mask dtypes / layouts / thresholds / thinning against the oracle:
    selected pixels, hypotheses (bit pattern), counts and winners exact, keypoints within 1e-4 px."""
    rng = np.random.default_rng(1000 + case)
    H, W = int(rng.integers(8, 160)), int(rng.integers(8, 200))
    K, hn, B = int(rng.integers(1, 7)), int(rng.integers(1, 320)), int(rng.integers(1, 4))
    fill = float(rng.uniform(0.05, 0.7))
    cfg = dict(B=B, H=H, W=W, K=K, hn=hn, fill=(fill, fill), kind=str(rng.choice(["blob", "fragmented"])))
    layout = str(rng.choice(["interleaved", "planar"]))
    mask, vertex, _ = _inputs(pvb, cfg, seed=2000 + case, layout=layout, noise_deg=float(rng.uniform(0, 8)),
                              outlier_frac=float(rng.uniform(0, 0.6)))
    dtype = [torch.int64, torch.int32, torch.uint8, torch.bool, torch.float32][int(rng.integers(0, 5))]
    fg = int(mask[0].sum())
    max_num = int(rng.choice([30000, max(6, fg // 2), max(6, fg // 5)]))
    thresh = float(rng.choice([0.99, 0.999, 0.95, 0.8]))
    _check_v3(pvb, oracle, mask.to(dtype), vertex, hn, thresh=thresh, seed=int(rng.integers(0, 2 ** 62)),
              img_base=int(rng.integers(0, 1000)), max_num=max_num, min_num=int(rng.integers(1, 9)))


def test_v3_seed_follows_torch_manual_seed(pvb):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=11)
    torch.manual_seed(5)
    a = pvb.ransac_voting_layer_v3(mask, vertex, 32, inlier_thresh=0.99)
    torch.manual_seed(5)
    b = pvb.ransac_voting_layer_v3(mask, vertex, 32, inlier_thresh=0.99)
    assert torch.equal(a, b)


def test_v1_alias(pvb):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=12)
    a = pvb.ransac_voting_layer(mask, vertex, 32, inlier_thresh=0.99, seed=3)
    b = pvb.ransac_voting_layer_v3(mask, vertex, 32, inlier_thresh=0.99, seed=3)
    assert torch.equal(a, b)


def test_distribution_matches_oracle(pvb, oracle):
    mask, vertex, kp = _inputs(pvb, "small", seed=13)
    mean = pvb.ransac_voting_layer_v3(mask, vertex, 64, inlier_thresh=0.99, seed=1)
    mean_out, cov, dbg = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=64,
                                                                    min_hyp_num=512, seed=77, debug=True)
    assert mean_out is mean
    m, v, mu = _np(mask, vertex, mean)
    _, want, odbg = oracle.estimate_voting_distribution_with_mean(m, v, mu, round_hyp_num=64, min_hyp_num=512,
                                                                  seed=77, debug=True)
    assert bits_equal(dbg["hyp"].cpu().numpy(), odbg["hyp"])
    tn = dbg["tn"].cpu().numpy().astype(np.float32)
    ratio = dbg["counts"].cpu().numpy().astype(np.float32) / tn[:, None, None]
    assert np.array_equal(ratio, odbg["ratio"])
    got = cov.cpu().numpy()
    assert got.shape == (mask.shape[0], vertex.shape[3], 2, 2)
    restated = check_covariance(cov, dbg, mean)
    assert np.allclose(want, restated, rtol=1e-6, atol=1e-9 * np.abs(restated).max())      # the oracle agrees
    assert np.array_equal(got[..., 0, 1], got[..., 1, 0])


def test_distribution_mask_equals_one_and_skip(pvb, oracle):
    """The distribution op selects mask == 1 only (:207) and returns ones/zeros for tiny foregrounds (:211-216)."""
    mask, vertex, _ = _inputs(pvb, "tiny", seed=14)
    m = mask.clone()
    m[1][mask[1] == 1] = 2        # class 2 only: no pixel equals 1 -> skipped
    mean = torch.rand((2, vertex.shape[3], 2), device="cuda") * 40
    _, cov, dbg = pvb.estimate_voting_distribution_with_mean(m, vertex, mean, round_hyp_num=32, min_hyp_num=128, seed=2,
                                                             debug=True)
    mn, vn_, mu = _np(m, vertex, mean)
    _, want, odbg = oracle.estimate_voting_distribution_with_mean(mn, vn_, mu, round_hyp_num=32, min_hyp_num=128, seed=2,
                                                                  debug=True)
    assert dbg["state"].tolist() == [0, 1] and bits_equal(dbg["hyp"].cpu().numpy(), odbg["hyp"])
    restated = check_covariance(cov, dbg, mean)
    assert np.allclose(want, restated, rtol=1e-6, atol=1e-9 * np.abs(restated).max())      # the oracle agrees
    exp = np.einsum("ki,kj->kij", mu[1], mu[1]) * 128 / (np.float32(128) + np.float32(1e-3))
    assert np.allclose(cov[1].cpu().numpy(), exp, rtol=1e-5)


def test_error_paths(pvb):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=15)
    with pytest.raises(RuntimeError, match="shape"):
        pvb.ransac_voting_layer_v3(mask, vertex, 32, idxs=torch.zeros(1, 2, 3, 2, dtype=torch.int32, device="cuda"))
    with pytest.raises(RuntimeError):
        pvb.ransac_voting_layer_v3(mask[:, :-1], vertex, 32)
    # a workspace too small for the adversarial selection is reported, not overrun
    B, H, W = mask.shape
    sel = torch.zeros((B, H, W), device="cuda")           # keeps every foreground pixel
    big = torch.ones_like(mask)
    with pytest.raises(RuntimeError, match="cannot hold"):          # refused on the host, before anything is launched
        pvb.ransac_voting_layer_v3(big, vertex, 32, max_num=100, selection=sel, capacity=256)
    # ... and if a caller of the C ABI gets it wrong anyway, the device reports it (sticky status), nothing is overrun
    from clean_pvnet_b200 import ransac_voting_gpu as op
    op._VALIDATE_CAPACITY = False
    try:
        with pytest.raises(RuntimeError, match="selected more than capacity"):
            pvb.ransac_voting_layer_v3(big, vertex, 32, max_num=100, selection=sel, capacity=256, debug=True)
    finally:
        op._VALIDATE_CAPACITY = True


def test_empty_batch_and_empty_foreground(pvb):
    mask, vertex, _ = _inputs(pvb, "tiny", seed=17)
    out = pvb.ransac_voting_layer_v3(mask[:0], vertex[:0], 32, inlier_thresh=0.99)
    assert out.shape == (0, vertex.shape[3], 2)
    _, cov = pvb.estimate_voting_distribution_with_mean(mask[:0], vertex[:0], out)
    assert cov.shape == (0, vertex.shape[3], 2, 2)
    zero = torch.zeros_like(mask)
    out = pvb.ransac_voting_layer_v3(zero, vertex, 32, inlier_thresh=0.99)
    assert (out == 0).all()                          # every image skipped (:129-132)
    one_px = zero.clone()
    one_px[:, 5, 5] = 1
    out = pvb.ransac_voting_layer_v3(one_px, vertex, 32, inlier_thresh=0.99, min_num=1)
    assert torch.isfinite(out).all()                 # tn == 1: every pair is degenerate -> hypotheses (0,0)


def test_cuda_graph_capture_and_replay(pvb):
    """The device entry points enqueue only (no sync, no allocation inside the library): one v3 +
    distribution call is captured into a CUDA graph and replayed on new input values."""
    mask, vertex, _ = _inputs(pvb, "small", seed=18)
    static_mask, static_vertex = mask.clone(), vertex.clone()
    want = pvb.ransac_voting_layer_v3(static_mask, static_vertex, 64, inlier_thresh=0.99, seed=9, max_num=800)
    _, want_cov = pvb.estimate_voting_distribution_with_mean(static_mask, static_vertex, want, round_hyp_num=64,
                                                             min_hyp_num=256, seed=10)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        # warm the per-stream workspace outside the capture
        pvb.ransac_voting_layer_v3(static_mask, static_vertex, 64, inlier_thresh=0.99, seed=9, max_num=800)
        pvb.estimate_voting_distribution_with_mean(static_mask, static_vertex, want, round_hyp_num=64, min_hyp_num=256, seed=10)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            out = pvb.ransac_voting_layer_v3(static_mask, static_vertex, 64, inlier_thresh=0.99, seed=9, max_num=800)
            _, cov = pvb.estimate_voting_distribution_with_mean(static_mask, static_vertex, out, round_hyp_num=64,
                                                                min_hyp_num=256, seed=10)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want) and torch.equal(cov, want_cov)
    # new data in the static buffers, replay only
    mask2, vertex2, _ = _inputs(pvb, "small", seed=19)
    static_mask.copy_(mask2); static_vertex.copy_(vertex2)
    g.replay()
    torch.cuda.synchronize()
    want2 = pvb.ransac_voting_layer_v3(mask2, vertex2, 64, inlier_thresh=0.99, seed=9, max_num=800)
    assert torch.equal(out, want2)


def test_host_buffer_entry_matches_device_entry(pvb):
    mask, vertex, _ = _inputs(pvb, "small", seed=16, B=5)
    dev = pvb.ransac_voting_layer_v3(mask, vertex, 64, inlier_thresh=0.99, seed=21, max_num=700)
    mh, vh = mask.cpu().pin_memory(), vertex.cpu().pin_memory()
    for chunk in (1, 2, 5):
        for mode in ("auto", "inplace", "staged"):   # mask by DMA + vertex rows in place / all in place / all copied
            host = pvb.ransac_voting_layer_v3_host(mh, vh, 64, inlier_thresh=0.99, seed=21, max_num=700,
                                                   chunk_images=chunk, mode=mode)
            assert not host.is_cuda
            assert torch.equal(host, dev.cpu())
    # pageable (unpinned) inputs silently take the staged path
    host = pvb.ransac_voting_layer_v3_host(mask.cpu(), vertex.cpu(), 64, inlier_thresh=0.99, seed=21, max_num=700)
    assert torch.equal(host, dev.cpu())


# ---- BASELINE.json full-size configuration: size-independent properties ---------------------
def test_full_size_noise_free_recovery(pvb):
    """cfg-2 shape (B=16, 480x640, K=9, hn=512): on a noise-free field every keypoint -- including the
    one outside the image -- is recovered; results are deterministic and shard-invariant."""
    mask, vertex, kp = _inputs(pvb, "cfg2", seed=1236, noise_deg=0.0, outlier_frac=0.0, B=4)
    out = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99, seed=5)
    assert (out - kp).abs().max().item() < 2e-2
    out2 = torch.cat([pvb.ransac_voting_layer_v3(mask[i:i + 1], vertex[i:i + 1], 512, inlier_thresh=0.99, seed=5,
                                                 img_base=i) for i in range(4)])
    assert torch.equal(out, out2)


def test_full_size_counts_against_reference_formulation(pvb):
    """cfg-2 shape: the fused counts equal the byte-tensor formulation of the reference
    (voting_for_hypothesis -> sum) evaluated with the exact-arithmetic twin kernel."""
    mask, vertex, _ = _inputs(pvb, "cfg2", seed=1240, B=1)
    _, dbg = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99, seed=8, debug=True)
    tn = int(dbg["tn"][0])
    assert abs(tn - 30000) < 1200
    direct = dbg["dirs"][0, :, :tn].permute(1, 0, 2).contiguous()       # [tn,K,2]
    coords = dbg["xy"][0, :tn].contiguous()
    hyp = dbg["hyp"][0].permute(1, 0, 2).contiguous()                    # [hn,K,2]
    K = direct.shape[1]
    for k0 in range(0, K, 3):
        inl = torch.zeros((512, 3, tn), dtype=torch.uint8, device="cuda")
        pvb.ransac_voting.voting_for_hypothesis(direct[:, k0:k0 + 3].contiguous(), coords,
                                                hyp[:, k0:k0 + 3].contiguous(), inl, 0.99)
        want = inl.sum(dim=2, dtype=torch.int32)                          # [hn,3]
        assert torch.equal(dbg["counts"][0, k0:k0 + 3].t().contiguous(), want)


def test_full_size_refit_normal_equations(pvb):
    """cfg-2 shape, B = 2 (~30 000 selected pixels = 15 refit CTAs per keypoint): the refit sums exactly the winner's
    inliers under the reference predicate, evaluated by the byte-tensor twin kernel."""
    mask, vertex, _ = _inputs(pvb, "cfg2", seed=1243, B=2)
    _, dbg = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99, seed=9, debug=True)
    tn = dbg["tn"].cpu().numpy()
    assert (np.abs(tn - 30000) < 1200).all()
    assert ((tn + 2047) // 2048 >= 14).all()
    cnt = check_normal_eq(dbg, 0.99, twin_inliers(pvb))
    assert (cnt > 1000).all()


@pytest.mark.parametrize("H,W,K,max_num,layout", [
    (48, 64, 3, 30000, "interleaved"),      # whole words, no thinning: every foreground pixel selected
    (37, 53, 4, 30000, "interleaved"),      # H*W = 1961: the image ends inside a bitmap word
    (37, 53, 5, 200, "interleaved"),        # thinned to ~200 of ~600
    (96, 128, 9, 150, "interleaved"),       # thinned hard
    (48, 64, 3, 30000, "planar"),           # strided NCHW view: the row-wise walk does not apply and falls back
])
def test_every_gather_walk_gives_the_same_compaction(pvb, H, W, K, max_num, layout):
    """The gather kernel's access patterns (include/pvnet_vote_b200.h, pvb_set_tuning gather_mode): pixel-wise, row-wise
    (what in-place host reads use) and the automatic choice must produce bit-identical xy / dirs / keypoints."""
    from clean_pvnet_b200 import _lib, synth
    lib = _lib.load()
    cfg = dict(B=3, H=H, W=W, K=K, hn=32, fill=(0.25, 0.4), kind="blob")
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=77, layout=layout)
    mask[2, H - 1, W - 3:] = 1                                   # foreground in the very last (partial) word
    ref = None
    try:
        for mode in (1, 2, 0):
            _lib.check(lib.pvb_set_tuning(mode, 0))
            out, dbg = pvb.ransac_voting_layer_v3(mask, vertex, 32, inlier_thresh=0.99, seed=5, max_num=max_num, debug=True)
            tn = dbg["tn"].tolist()                               # entries past tn are never written by any walk
            got = (out, dbg["tn"], dbg["counts"]) + tuple(dbg["xy"][b, :tn[b]] for b in range(3)) + \
                tuple(dbg["dirs"][b, :, :tn[b]] for b in range(3))
            if ref is None:
                ref = got
                assert int(dbg["tn"].min()) > 0
            else:
                for a, b in zip(ref, got):
                    assert torch.equal(a, b), mode
    finally:
        _lib.check(lib.pvb_set_tuning(0, 0))
