"""GPU tests of each batched op at the capacity its C ABI accepts (tests/limits.py), where staging loops take a second
pass, lists reach their cap and launches split.  Each case is compared with the restatement the op's own GPU tests
trust:
  - ct_focal_loss / ct_target_batch at M = 256, 257 and 1024 objects per image, C = 30 and C = 1 with every object in
    one tile: the target bit for bit, the gradient equal to autograd's bit for bit, the loss within 1e-5;
  - vote_loss / vote_target_batch at K = 256, 257 and 1024 keypoints: the same three bars, the loss within one fp32 ulp
    of the chain on a float64 sum;
  - instance_masks_from_depth at 256, 257 and 2048 instances in one image and a batch of 2048, 1 and 257: bit for bit;
  - decode_detections at K = 1024, 1025, 4096 and H*W on plateaus and noisy blobs: bit for bit against the stable-sort
    restatement, as sets on tied rows against the two-topk one;
  - ransac_voting_layer_v3 at hn = 2048 with K = 2047 (pruned), 2048 (not pruned) and 16383 (the ABI's largest), and
    estimate_voting_distribution_with_mean at K = 16383: keypoints spread over the range equal a K = 1 call bit for bit,
    and match the CPU oracle;
  - render_depth_batch of 3300 poses of an icosphere(5), two launches: poses on both sides of the split equal a
    single-pose render bit for bit, with a shared and a per-pose K, and match the fp64 oracle.
Every case's peak device memory stays within limits.DEVICE_BUDGET."""
import numpy as np
import pytest
import torch

import ct_decode_cases as dc
import limits as lm
from ct_target_cases import restate_batch
from tless_mask_cases import _blob, _same_key_pair, _surface, compose_restated
from vote_target_cases import restate_vertex

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


class _Peak:
    """Peak device memory allocated inside the block, over what was allocated when it began."""

    def __enter__(self):
        torch.cuda.synchronize()
        self.start = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.bytes = torch.cuda.max_memory_allocated() - self.start
        return False

    def check(self, label, estimate):
        print(f"[limits] {label}: peak {self.bytes / 2 ** 20:.0f} MiB (estimate {estimate / 2 ** 20:.0f} MiB)")
        assert self.bytes <= lm.DEVICE_BUDGET, label


def _bits_equal(a, b):
    """Equal bit for bit, except that any NaN equals any NaN."""
    a, b = a.detach(), b.detach()
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    return torch.equal(a[~na].contiguous().view(torch.int32), b[~nb].contiguous().view(torch.int32))


def _ulps(a, b):
    return abs(int(np.array([a], np.float32).view(np.int32)[0]) - int(np.array([b], np.float32).view(np.int32)[0]))


# ---- ct_focal_loss ----------------------------------------------------------------------------------------------------

def _ct_objects(M, C, seed):
    """[B,M] objects, every row real except a few padding rows of image 3 (garbage values, ct_01 = 0), none of them the
    last.  C = 1: the centres are a random permutation of one 32x16 tile's pixels (repeating past 512), so each of the
    first 512 objects has a centre of its own and every window meets that tile."""
    B, H, W = lm.CT_SHAPE["B"], lm.CT_SHAPE["H"], lm.CT_SHAPE["W"]
    rng = np.random.default_rng(seed)
    if C == 1:
        tw, th = lm.CT_TILE
        x0, y0 = tw, th                                   # the tile in the second column and row
        pos = np.concatenate([np.stack([rng.permutation(tw * th) for _ in range(B)]),
                              rng.integers(0, tw * th, (B, max(0, M - tw * th)))], 1)[:, :M]
        ind = ((y0 + pos // tw) * W + x0 + pos % tw).astype(np.int64)
        rad = rng.integers(0, 13, (B, M)).astype(np.int32)
    else:
        ind = rng.integers(0, H * W, (B, M)).astype(np.int64)
        rad = rng.integers(0, 20, (B, M)).astype(np.int32)
    cls = rng.integers(0, C, (B, M)).astype(np.int64)
    c01 = np.ones((B, M), np.float32)
    pad = rng.choice(M - 1, 5, replace=False)
    c01[3, pad] = 0
    ind[3, pad[:2]], cls[3, pad[2:4]], rad[3, pad[4]] = H * W + 7, C + 2, -3
    return ind, rad, cls, c01


@pytest.mark.parametrize("C", lm.CT_SHAPE["C"])
@pytest.mark.parametrize("M", lm.CT_LOSS.cases)
def test_ct_loss_at_capacity(pvb, M, C):
    from test_gpu_ct_loss import _logits, _reference_loss
    B, H, W = lm.CT_SHAPE["B"], lm.CT_SHAPE["H"], lm.CT_SHAPE["W"]
    ind, rad, cls, c01 = _ct_objects(M, C, seed=M * 100 + C)
    want = restate_batch(ind, rad, cls, c01, C, H, W)
    if C == 1:                                            # every object's own centre is a peak of 1
        assert ((want[:3, 0] == 1).sum(axis=(1, 2)) == min(M, 512)).all()
    with _Peak() as peak:
        objs = [torch.from_numpy(a).to(DEV) for a in (ind, rad, cls, c01)]
        assert torch.equal(pvb.ct_target_batch(*objs, C, H, W), torch.from_numpy(want).to(DEV))
        dense = torch.from_numpy(want).to(DEV)
        x = _logits(B, C, H, W, seed=M + C)
        a = x.clone().requires_grad_()
        ref = _reference_loss(a, dense)
        (ref * 1.5).backward()
        b = x.clone().requires_grad_()
        got = pvb.ct_focal_loss(b, *objs)
        (got * 1.5).backward()
        assert _bits_equal(b.grad, a.grad)
        r, g = float(ref.detach()), float(got.detach())
        assert abs(g - r) <= 1e-5 * abs(r), (g, r)
    peak.check(f"ct M={M} C={C}", lm.ct_bytes(M, C))


# ---- vote_loss --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mask_dtype", [torch.uint8, torch.int64, torch.bool])
@pytest.mark.parametrize("K", lm.VOTE_LOSS.cases)
def test_vote_loss_at_capacity(pvb, K, mask_dtype):
    from test_gpu_vote_loss import _grads, _inputs, _pred
    B, H, W = lm.VOTE_LOSS_SHAPE["B"], lm.VOTE_LOSS_SHAPE["H"], lm.VOTE_LOSS_SHAPE["W"]
    mask_np, kpt_np = _inputs(B, H, W, K, seed=K, fill=0.35, values=(1, 1, 1, 2, 255))
    if mask_dtype == torch.bool:
        mask_np = mask_np != 0
    want = np.stack([restate_vertex(m, k) for m, k in zip(mask_np, kpt_np)])
    with _Peak() as peak:
        mask = torch.from_numpy(mask_np).to(DEV).to(mask_dtype)
        kpt = torch.from_numpy(kpt_np).to(DEV)
        vertex = torch.from_numpy(want).to(DEV)
        assert _bits_equal(pvb.vote_target_batch(mask, kpt), vertex)
        leaf, view = _pred(B, K, H, W, seed=K + 1, layout="contiguous")
        _, _, gref, ggot = _grads(pvb, leaf, view, mask, kpt, vertex, -0.7)
        assert _bits_equal(ggot, gref)
        del gref, ggot, leaf
        # the forward against the same chain on a float64 sum of the terms, one image at a time
        pred = view(torch.randn(B, 2 * K, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(K)))
        loss = float(pvb.vote_loss(pred, mask, kpt))
        s64 = 0.0
        for b in range(B):
            w = mask[b, None].float()
            x = (pred[b] * w - vertex[b] * w).double()
            ax = x.abs()
            s64 += float(torch.where(ax < 1, 0.5 * x * x, ax - 0.5).sum())
        wsum = np.float32(float(mask.to(torch.int64).sum()))
        fp64 = np.float32(np.float32(np.float32(s64) / wsum) * (np.float32(1) / np.float32(2 * K)))
        assert _ulps(loss, fp64) <= 1, (loss, fp64)
    peak.check(f"vote_loss K={K} {mask_dtype}", lm.vote_loss_bytes(K))


# ---- instance masks ---------------------------------------------------------------------------------------------------

NEAR = 8                                                   # slots of small near blobs, kept for late instances


def _mask_slots(rng):
    """[S,H,W] depth slots in mm: an empty one, the far plane, a same-key pair, an equal-depth pair, random tilted
    blobs on a 0.5 mm grid (so reuses tie), and NEAR small blobs at 300 mm that no earlier slot can hide."""
    H, W, S = lm.MASK_SHAPE["H"], lm.MASK_SHAPE["W"], lm.MASK_SHAPE["slots"]
    d = np.zeros((S, H, W), np.float32)
    d[1] = 10000.0
    k0, k1 = _same_key_pair(rng)
    d[2, 3:40, 3:50], d[3, 20:60, 30:80] = k1, k0
    d[4, 10:50, 10:40] = d[5, 30:61, 20:70] = 800.0
    for s in range(6, S - NEAR):
        m = _blob(rng, H, W)
        d[s][m] = _surface(rng, H, W)[m]
    for i in range(NEAR):
        y, x = 4 + 7 * i, 5 + 9 * i
        d[S - NEAR + i, y:y + 5, x:x + 6] = 300.0 + i
    return d


def _mask_instances(m, rng):
    """Slot and obj_id of each of m instances: random slots, and the NEAR slots only at late positions (the flush's
    second and later passes, and the last instance), obj_id 30 there."""
    S = lm.MASK_SHAPE["slots"]
    slot = rng.integers(0, S - NEAR, m)
    obj = rng.integers(1, lm.MAX_OBJ_ID + 1, m)
    late = sorted({j for j in (m - 1, m - 2, lm.MASKS.stride, lm.MASKS.stride + 1, m // 2, 3 * m // 4, 2 * lm.MASKS.stride)
                   if 0 <= j < m})[:NEAR]
    slot[late] = S - NEAR + np.arange(len(late))
    obj[late] = lm.MAX_OBJ_ID
    return slot, obj, late


@pytest.mark.parametrize("counts", [(256,), (257,), (2048,), lm.MASK_BATCH], ids=["256", "257", "2048", "batch"])
def test_instance_masks_at_capacity(pvb, counts):
    from test_gpu_tless_masks import assert_equal
    rng = np.random.default_rng(sum(counts))
    depth = _mask_slots(rng)
    H, W = lm.MASK_SHAPE["H"], lm.MASK_SHAPE["W"]
    slots, objs, image_index, lates = [], [], [], []
    for b, m in enumerate(counts):
        s, o, late = _mask_instances(m, rng)
        lates += [sum(counts[:b]) + j for j in late]
        slots.append(s), objs.append(o), image_index.append(np.full(m, b))
    slot, obj, img = np.concatenate(slots), np.concatenate(objs), np.concatenate(image_index)
    label = np.zeros((len(counts), H, W), np.int16)
    a, p, bb = np.zeros(len(img), np.int64), np.zeros(len(img), np.int64), np.zeros((len(img), 4), np.int64)
    for b in range(len(counts)):
        idx = np.flatnonzero(img == b)
        label[b], a[idx], p[idx], bb[idx] = compose_restated(depth[slot[idx]], obj[idx])
    assert (p[lates] > 0).all()                          # every late instance takes pixels
    assert label.max() == lm.MAX_OBJ_ID * 1000 + max(counts) - 1     # 32047 at 2048 instances
    with _Peak() as peak:
        got = pvb.instance_masks_from_depth(torch.from_numpy(depth).to(DEV), slot, obj, img)
        assert_equal(got, (label, a, p, bb))
    peak.check(f"masks {counts}", lm.mask_bytes(counts))


# ---- decode -----------------------------------------------------------------------------------------------------------

def _decode_logits(kind, rng, C):
    """'blobs': noisy blobs.  'plateau': noisy blobs below 1, each class's first 32x32 tile at logit 30 (sigmoid exactly
    1, so that one tile holds the top 1024 keys of its class), a patch of +inf inside it, a -inf region (exact zeros)
    and two rows at -30 (one tiny value)."""
    B, H, W = lm.DECODE_SHAPE["B"], lm.DECODE_SHAPE["H"], lm.DECODE_SHAPE["W"]
    lg = dc.blobs(rng, B, C, H, W, noise=0.3)
    if kind == "plateau":
        lg[:, :, :lm.DECODE_TILE, :lm.DECODE_TILE] = 30.0
        lg[:, :, 5:9, 5:9] = np.inf
        lg[:, :, 40:60, 40:80] = -np.inf
        lg[:, :, 70:72, :] = -30.0
    return torch.from_numpy(lg).to(DEV), torch.from_numpy(dc._wh(rng, B, H, W)).to(DEV)


def _bits(t):
    t = t.detach().float().cpu().contiguous()
    return torch.where(t.isnan(), torch.full_like(t, float("nan")), t).view(torch.int32).numpy()


def _same_as_sets(det, ct, want_det, want_ct):
    """Against the two-topk restatement: the score column bit for bit; the rows outside the group of scores the K-th
    row ends in, as one multiset per image (a row holds its score, so this compares each tied group as a set)."""
    assert np.array_equal(_bits(det[..., 4]), _bits(want_det[..., 4]))
    rows, want = _bits(torch.cat([det, ct], -1)), _bits(torch.cat([want_det, want_ct], -1))
    for b in range(rows.shape[0]):
        keep = rows[b, :, 4] != rows[b, -1, 4]
        r, w = rows[b][keep], want[b][keep]
        assert np.array_equal(r[np.lexsort(r.T[::-1])], w[np.lexsort(w.T[::-1])]), b


@pytest.mark.parametrize("kind", ["plateau", "blobs"])
@pytest.mark.parametrize("K", lm.DECODE.cases)
def test_decode_at_capacity(pvb, K, kind):
    H, W = lm.DECODE_SHAPE["H"], lm.DECODE_SHAPE["W"]
    C = 1 if K == H * W else lm.DECODE_SHAPE["C"][0]
    rng = np.random.default_rng(K + len(kind))
    with _Peak() as peak:
        lg, wh = _decode_logits(kind, rng, C)
        for clip in (True, False):
            ct, det = pvb.decode_detections(lg, wh, K, clip)
            want_ct, want_det = dc.restate_decode_ordered(lg, wh, K, clip)
            assert np.array_equal(_bits(ct), _bits(want_ct)), clip
            bad = (_bits(det) != _bits(want_det)).any(-1).nonzero()
            assert bad[0].size == 0, (clip, list(zip(*bad))[:8])
            topk_ct, topk_det = dc.restate_decode(lg, wh, K, clip)
            _same_as_sets(det, ct, topk_det, topk_ct)
        if kind == "plateau":                             # the top 1024 keys of each class lie in its first tile
            s = det[:, :min(K, 1024), 4]
            assert bool((s == 1).all())
    peak.check(f"decode K={K} {kind}", lm.decode_bytes(K, C))


def test_decode_every_key_time(pvb):
    """K = H*W on the training map: the select kernel ranks all 13312 keys in one CTA per image.  Prints the time."""
    H, W = lm.DECODE_SHAPE["H"], lm.DECODE_SHAPE["W"]
    lg, wh = _decode_logits("blobs", np.random.default_rng(3), 1)
    pvb.decode_detections(lg, wh, H * W)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 5
    e0.record()
    for _ in range(n):
        pvb.decode_detections(lg, wh, H * W)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(f"[limits] decode_detections B=2 C=1 {H}x{W} K={H * W}: {ms:.3f} ms per call on {torch.cuda.get_device_name()}")
    assert ms < 1000


# ---- the vote layer ---------------------------------------------------------------------------------------------------

THRESH = 0.99


def _vote_inputs(K, seed):
    """A full mask on a tiny image, a noisy field towards one random target per keypoint (a fifth of the pixels
    random), and explicit sample pairs.  The field is made on the host, so no temporaries of its size hit the device."""
    B, H, W = lm.VOTE_LAYER_SHAPE["B"][K], lm.VOTE_LAYER_SHAPE["H"], lm.VOTE_LAYER_SHAPE["W"]
    rng = np.random.default_rng(seed)
    tgt = rng.uniform((-W, -H), (2 * W, 2 * H), (B, 1, 1, K, 2)).astype(np.float32)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float32)
    ang = np.arctan2(tgt[..., 1] - ys[None, :, :, None], tgt[..., 0] - xs[None, :, :, None])
    ang += rng.normal(0, np.radians(3), ang.shape).astype(np.float32)
    out = rng.random(ang.shape) < 0.2
    ang[out] = rng.uniform(0, 2 * np.pi, int(out.sum()))
    vertex = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)
    mask = torch.ones((B, H, W), dtype=torch.uint8, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    idxs = torch.randint(0, H * W, (B, lm.VOTE_LAYER_HN, K, 2), generator=g, device=DEV, dtype=torch.int32)
    return mask, torch.from_numpy(vertex).to(DEV), idxs


def _check_keypoints(pvb, oracle, mask, vertex, idxs, out, K):
    """out[:, k] equals a K = 1 call on keypoint k's field and sample pairs bit for bit, and that call matches the CPU
    oracle: hypotheses bit for bit, counts and winner exactly, keypoint within 1e-4 px."""
    hn = lm.VOTE_LAYER_HN
    m = mask.cpu().numpy().astype(np.int64)
    for k in lm.vote_keypoints(K):
        v1, i1 = vertex[..., k:k + 1, :], idxs[..., k:k + 1, :]
        one = pvb.ransac_voting_layer_v3(mask, v1, hn, inlier_thresh=THRESH, idxs=i1, seed=0)
        assert _bits_equal(out[:, k:k + 1], one), k
        dbg_out, dbg = pvb.ransac_voting_layer_v3(mask, v1, hn, inlier_thresh=THRESH, idxs=i1, seed=0, debug=True)
        assert _bits_equal(dbg_out, one), k
        want, odbg = oracle.ransac_voting_layer_v3(m, v1.cpu().numpy(), hn, inlier_thresh=THRESH,
                                                   idxs=i1.cpu().numpy(), debug=True)
        assert np.array_equal(dbg["hyp"].cpu().numpy().view(np.int32), odbg["hyp"].view(np.int32)), k
        assert np.array_equal(dbg["counts"].cpu().numpy(), odbg["counts"]), k
        assert np.array_equal(dbg["win"].cpu().numpy().view(np.int32), odbg["win"].view(np.int32)), k
        assert np.abs(one.cpu().numpy() - want).max() < 1e-4, k


@pytest.mark.parametrize("K", lm.VOTE_LAYER.cases[:2])
def test_vote_layer_at_the_prune_gate(pvb, oracle, K):
    from prune_twin import prune_applies
    from test_gpu_prune import _compare
    with _Peak() as peak:
        mask, vertex, idxs = _vote_inputs(K, seed=K)
        B = mask.shape[0]
        out = pvb.ransac_voting_layer_v3(mask, vertex, lm.VOTE_LAYER_HN, inlier_thresh=THRESH, idxs=idxs, seed=0)
        assert prune_applies(THRESH, lm.VOTE_LAYER_HN, B, K) == (K == lm.VOTE_LAYER.cases[0])
        if K == lm.VOTE_LAYER.cases[0]:                   # the pruned call equals the full path, hypothesis by hypothesis
            _compare(pvb, mask, vertex, lm.VOTE_LAYER_HN, THRESH, idxs=idxs, seed=0)
        _check_keypoints(pvb, oracle, mask, vertex, idxs, out, K)
    peak.check(f"vote layer K={K}", lm.vote_layer_bytes(K))


def test_vote_layer_and_distribution_at_the_abi_limit(pvb, oracle):
    from clean_pvnet_b200 import ransac_voting_gpu as rv
    K = lm.VOTE_LAYER.cases[-1]
    hn = lm.VOTE_LAYER_HN
    try:
        with _Peak() as peak:
            mask, vertex, idxs = _vote_inputs(K, seed=K)
            out = pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=THRESH, idxs=idxs, seed=0)
            _check_keypoints(pvb, oracle, mask, vertex, idxs, out, K)
            _, cov = pvb.estimate_voting_distribution_with_mean(mask, vertex, out, round_hyp_num=lm.DIST_ROUND_HN,
                                                                min_hyp_num=hn, idxs=idxs, seed=0)
            assert torch.isfinite(cov).all()
            for k in lm.vote_keypoints(K):
                _, one = pvb.estimate_voting_distribution_with_mean(
                    mask, vertex[..., k:k + 1, :], out[:, k:k + 1], round_hyp_num=lm.DIST_ROUND_HN, min_hyp_num=hn,
                    idxs=idxs[..., k:k + 1, :], seed=0)
                assert _bits_equal(cov[:, k:k + 1], one), k
            del vertex, idxs
        peak.check(f"vote layer K={K}", lm.vote_layer_bytes(K))
    finally:
        rv._workspaces.clear()                            # gives back the gigabyte this call's workspace holds
        torch.cuda.empty_cache()


# ---- render -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("per_k", [False, True], ids=["sharedK", "poseK"])
def test_render_across_the_launch_split(pvb, per_k):
    import render_oracle
    from test_gpu_render import compare_with_oracle, per_pose_k
    from vsd_cases import K_SMALL, icosphere, poses
    render_oracle.build()
    v, f = icosphere(lm.RENDER_SUBDIV)
    assert len(f) == lm.RENDER_FACES
    n = lm.RENDER.cases[0]
    P = poses(n, seed=17)
    K0 = K_SMALL.copy()
    K0[0, 2], K0[1, 2] = lm.RENDER_SIZE[0] / 2 - 0.3, lm.RENDER_SIZE[1] / 2 + 0.1
    Ks = per_pose_k(K0, n, seed=5) if per_k else K0
    with _Peak() as peak:
        vd, fd = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
        depth = pvb.render_depth_batch(vd, fd, torch.from_numpy(P).to(DEV), torch.from_numpy(Ks).to(DEV), lm.RENDER_SIZE)
        for i in lm.RENDER_POSES:
            Ki = Ks[i] if per_k else K0
            one = pvb.render_depth_batch(vd, fd, P[i:i + 1], Ki, lm.RENDER_SIZE)
            assert torch.equal(depth[i], one[0]), i
            assert int((one[0] > 0).sum()) > 50, i
        d = depth[[lm.RENDER_POSES[1], lm.RENDER_POSES[2]]].cpu().numpy()
    for j, i in enumerate(lm.RENDER_POSES[1:3]):
        compare_with_oracle(d[j], v, f, P[i], Ks[i] if per_k else K0, lm.RENDER_SIZE, f"icosphere(5) n={n} pose {i}")
    peak.check(f"render n={n}", lm.render_bytes())
