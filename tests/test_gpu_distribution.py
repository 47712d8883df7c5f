"""GPU: the distribution stage -- estimate_voting_distribution_with_mean's selection (mask == 1, philox thinning tag 4),
hypotheses, ratios and covariance_kernel -- against the CPU oracle and a float64 restatement of the covariance.

Bars: tn, xy, hypotheses and ratios bit for bit; covariance entries within 1 fp32 ulp of the float64 restatement
(tests/util.py restated_covariance) plus 1e-12 * sum|terms| / den for off-diagonals that cancel."""
import numpy as np
import pytest
import torch

from util import bits_equal, check_covariance, restated_covariance

pytestmark = pytest.mark.gpu


def _inputs(cfg, seed, **kw):
    from clean_pvnet_b200 import synth
    return synth.make_inputs(cfg, device="cuda", seed=seed, **kw)


def _oracle_selection(oracle, mask, **kw):
    return oracle.select_pixels((mask.cpu() == 1).long().numpy(), 1, **kw)


def _idxs_for(tn, hn, K, seed):
    """Explicit sample pairs [B,hn,K,2] in [0, tn_b) per image (zeros for skipped or empty images)."""
    g = torch.Generator().manual_seed(seed)
    out = torch.zeros((len(tn), hn, K, 2), dtype=torch.int32)
    for b, t in enumerate(tn):
        if t > 0:
            out[b] = torch.randint(0, int(t), (hn, K, 2), generator=g, dtype=torch.int32)
    return out.cuda()


def _check_against_oracle(oracle, mask, vertex, mean, dbg, cov, rhn, mhn, **kw):
    """tn, xy, hypotheses and ratios equal the oracle's distribution operator bit for bit; the covariance passes the
    restatement bar."""
    m, v, mu = (t.cpu().numpy() for t in (mask, vertex, mean))
    okw = {k: (kw[k].cpu().numpy() if isinstance(kw[k], torch.Tensor) else kw[k]) for k in kw}
    _, want, odbg = oracle.estimate_voting_distribution_with_mean(m, v, mu, rhn, mhn, debug=True, **okw)
    sel = _oracle_selection(oracle, mask, **{k: okw[k] for k in ("selection", "seed", "min_num", "max_num") if k in okw})
    tn = dbg["tn"].cpu().numpy()
    assert np.array_equal(tn, np.maximum(sel["tn"], 0))
    W = mask.shape[2]
    for b, pix in enumerate(sel["pix"]):
        xy = np.stack([pix % W, pix // W], 1).astype(np.float32)
        assert bits_equal(dbg["xy"][b, :len(pix)].cpu().numpy(), xy)
    assert bits_equal(dbg["hyp"].cpu().numpy(), odbg["hyp"])
    live = dbg["state"].cpu().numpy() == 0
    with np.errstate(all="ignore"):
        ratio = dbg["counts"].cpu().numpy().astype(np.float32) / tn.astype(np.float32)[:, None, None]
    assert np.array_equal(ratio[live], odbg["ratio"][live], equal_nan=True)        # NaN: an image thinned to 0 pixels
    check_covariance(cov, dbg, mean)
    return want


def test_dist_thinning_matches_oracle_philox_and_explicit(pvb, oracle):
    """Thinned images (max_num below every foreground): the op's own philox stream (tag 4), then explicit `idxs` and
    explicit `selection`."""
    mask, vertex, kp = _inputs("small", 2101)
    mean = kp + 0.5
    kw = dict(max_num=700)
    _, cov, dbg = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, 64, 512, seed=31, debug=True, **kw)
    assert (dbg["nz"].cpu() > 700).all() and (dbg["tn"].cpu() < dbg["nz"].cpu()).all()
    _check_against_oracle(oracle, mask, vertex, mean, dbg, cov, 64, 512, seed=31, **kw)
    B, H, W = mask.shape
    selection = torch.rand((B, H, W), generator=torch.Generator(device="cuda").manual_seed(4), device="cuda")
    tn = _oracle_selection(oracle, mask, selection=selection.cpu().numpy(), **kw)["tn"]
    idxs = _idxs_for(tn, 512, vertex.shape[3], 5)
    _, cov, dbg = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, 64, 512, idxs=idxs, selection=selection,
                                                             debug=True, **kw)
    _check_against_oracle(oracle, mask, vertex, mean, dbg, cov, 64, 512, idxs=idxs, selection=selection, **kw)


@pytest.mark.parametrize("cfg,B", [("cfg2", 16), ("cfg4", 8)])
def test_full_size_default_arguments(pvb, oracle, cfg, B):
    """Default round_hyp_num 256 / min_hyp_num 4096 at full size.  The restatement trusts the op's hyp and counts, so
    those are checked first: hypotheses bit-equal to the oracle's generate_hypothesis for explicit idxs, counts equal to
    the oracle's vote_count on a random 256-hypothesis subset per (image, keypoint)."""
    mask, vertex, kp = _inputs(cfg, 2200 + B, B=B)
    _, H, W, K, _ = vertex.shape
    sel = _oracle_selection(oracle, mask, seed=41)                          # the op's philox thinning, tag 4
    idxs = _idxs_for(sel["tn"], 4096, K, 6)
    _, cov, dbg = pvb.estimate_voting_distribution_with_mean(mask, vertex, kp, idxs=idxs, seed=41, debug=True)
    assert np.array_equal(dbg["tn"].cpu().numpy(), sel["tn"]) and (sel["tn"] > 25000).all()
    vh = vertex.cpu().numpy()
    ih, hyp, counts = idxs.cpu().numpy(), dbg["hyp"].cpu().numpy(), dbg["counts"].cpu().numpy()
    rng = np.random.default_rng(B)
    for b in range(B):
        pix = sel["pix"][b].astype(np.int64)
        coords = np.stack([pix % W, pix // W], 1).astype(np.float32)
        direct = np.ascontiguousarray(vh[b].reshape(-1, K, 2)[pix])
        want = oracle.generate_hypothesis(direct, coords, ih[b])            # [hn,K,2]
        assert bits_equal(hyp[b], want.transpose(1, 0, 2)), b
        sub = np.stack([rng.choice(4096, 256, replace=False) for _ in range(K)], 1)       # [256,K]
        hs = np.ascontiguousarray(want[sub, np.arange(K)[None, :]])                       # [256,K,2]
        assert np.array_equal(oracle.vote_count(direct, coords, hs, 0.99), counts[b][np.arange(K)[None, :], sub]), b
    check_covariance(cov, dbg, kp)


@pytest.mark.parametrize("rhn,mhn", [(1, 1), (31, 31), (255, 255), (257, 257), (100, 250), (1024, 8192)])
def test_hypothesis_counts(pvb, oracle, rhn, mhn):
    """hn_total = round_hyp_num * ceil(min_hyp_num / round_hyp_num) of 1, 31, 255, 257, 300 and 8192 hypotheses: one
    partial warp up to 32 strided rounds per thread of the covariance kernel."""
    mask, vertex, kp = _inputs("small", 2300 + rhn)
    mean = kp - 2.0
    _, cov, dbg = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, rhn, mhn, seed=rhn, debug=True)
    assert dbg["hyp"].shape[2] == rhn * -(-mhn // rhn)
    _check_against_oracle(oracle, mask, vertex, mean, dbg, cov, rhn, mhn, seed=rhn)


def test_mixed_batch_and_far_mean(pvb, oracle):
    """One batch with a skipped image, a thinned one, an unthinned one and one thinned to zero pixels (NaN covariance,
    like the reference's 0/0 ratios); then the same with a mean 1e4 px away."""
    mask, vertex, kp = _inputs("small", 2400, B=4)
    B, H, W = mask.shape
    mask[0] = 0
    mask[0, 2, 3:7] = 1                                                     # 4 < min_num: skipped
    mask[2].view(-1)[torch.nonzero(mask[2].reshape(-1))[600:, 0]] = 0       # 600 pixels: below max_num
    selection = torch.rand((B, H, W), generator=torch.Generator(device="cuda").manual_seed(8), device="cuda")
    selection[3] = 0.99999                                                  # drops every pixel of image 3
    kw = dict(max_num=800, selection=selection)
    for mean in (kp + 1.5, kp + 1e4):
        _, cov, dbg = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, 128, 512, seed=9, debug=True, **kw)
        tn, nz, state = (dbg[k].cpu().numpy() for k in ("tn", "nz", "state"))
        assert state.tolist() == [1, 0, 0, 0] and tn[1] < nz[1] and tn[2] == nz[2] == 600 and tn[3] == 0 < nz[3]
        want = _check_against_oracle(oracle, mask, vertex, mean, dbg, cov, 128, 512, seed=9, **kw)
        assert torch.isnan(cov[3]).all() and np.isnan(want[3]).all() and torch.isfinite(cov[:3]).all()


def test_threshold_ties_are_kept(pvb, oracle):
    """Masks of exactly 10 and 20 foreground pixels, 4096 hypotheses: ratios land exactly on th = fp32(max - 0.1f)
    (e.g. 9/10 == fp32(1 - 0.1f), while the same threshold in float64 lies above 0.9f).  The reference keeps them
    (`ratio < th` is strict): ties occur, and dropping them would move the covariance far outside the bar."""
    for n in (10, 20):
        cfg = dict(B=2, H=32, W=48, K=3, hn=64, fill=(0.3, 0.3), kind="blob")
        from clean_pvnet_b200 import synth
        mask, vertex, kp = synth.make_inputs(cfg, device="cpu", seed=1, noise_deg=2.0, outlier_frac=0.1)
        g = torch.Generator().manual_seed(1)
        m = torch.zeros_like(mask)
        for b in range(2):
            on = torch.nonzero(mask[b].reshape(-1))[:, 0]
            m[b].view(-1)[on[torch.randperm(len(on), generator=g)[:n]]] = 1
        m, vertex, kp = m.cuda(), vertex.cuda(), kp.cuda()
        _, cov, dbg = pvb.estimate_voting_distribution_with_mean(m, vertex, kp, 256, 4096, seed=3, debug=True)
        assert (dbg["tn"].cpu() == n).all()
        ratio = dbg["counts"].cpu().numpy().astype(np.float32) / np.float32(n)
        th = (ratio.max(2) - np.float32(0.1)).astype(np.float32)
        ties = ratio == th[..., None]
        assert ties.sum() > 100
        th64 = ratio.max(2).astype(np.float64) - np.float64(np.float32(0.1))            # the threshold in float64
        assert (ratio.astype(np.float64) < th64[..., None])[ties].any()                  # ... would drop some ties
        want = check_covariance(cov, dbg, kp)
        _check_against_oracle(oracle, m, vertex, kp, dbg, cov, 256, 4096, seed=3)
        # the same sums without the tied hypotheses: some (image, keypoint) must then miss the bar
        d2 = dict(dbg)
        d2["counts"] = torch.from_numpy(np.where(ties, 0, dbg["counts"].cpu().numpy()))
        dropped, _ = restated_covariance(d2, kp)
        moved = np.abs(dropped - want) > np.spacing(np.abs(want).astype(np.float32)) * 4
        assert moved[ties.any(2)].any()


def test_skipped_images_with_partial_last_round(pvb):
    """min_hyp_num not a multiple of round_hyp_num (250 / 100 -> 300 hypotheses).  For a skipped image the reference
    builds min_hyp_num (250) unit ratios, this op hn_total (300) -- the reference can only run such a batch when every
    image is skipped (otherwise its torch.cat of 250- and 300-row blocks fails).  Pinned: cov = mean mean^T * 300 /
    fp32(300 + 1e-3f), which is a few ulp from the reference's 250 / fp32(250 + 1e-3f) (DESIGN.md)."""
    mask, vertex, _ = _inputs("tiny", 2500)
    mask.zero_()
    mean = torch.tensor([[[12.5, -3.25], [700.0, 0.1], [1e-3, 5.0]]] * 2, device="cuda")
    _, cov, dbg = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, 100, 250, seed=1, debug=True)
    assert dbg["hyp"].shape[2] == 300
    check_covariance(cov, dbg, mean)
    mu = mean.cpu().numpy().astype(np.float64)
    outer = mu[..., :, None] * mu[..., None, :]
    ours = (outer * 300 / np.float64(np.float32(300) + np.float32(1e-3))).astype(np.float32)
    ref = (outer * 250 / np.float64(np.float32(250) + np.float32(1e-3))).astype(np.float32)
    got = cov.cpu().numpy()
    assert np.array_equal(got, ours)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
    assert (ulps >= 4).all() and (ulps <= 12).all()          # relative 1e-3 * (1/250 - 1/300) = 6.7e-7
