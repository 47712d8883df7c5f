"""CPU tests of tests/limits.py: every capacity it states equals the constant in the source that enforces it, every case
tests/test_gpu_limits.py runs lies on the side of its boundary the table says, and every case fits the device-memory
and CPU-restatement budgets."""
import os
import re
import time

import numpy as np
import torch

import limits as lm
from prune_twin import prune_applies

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _src(path):
    with open(os.path.join(ROOT, path)) as f:
        return f.read()


def _const(path, name):
    m = re.findall(rf"^constexpr int (?:\w+ = \d+, )*{name} = (\d+)[;,]", _src(path), re.M)
    assert len(m) == 1, (path, name, m)
    return int(m[0])


# ---- the constants ----------------------------------------------------------------------------------------------------

def test_ct_loss_constants():
    path = lm.CT_LOSS.source
    assert _const(path, "CT_MAX_M") == lm.CT_LOSS.value
    assert _const(path, "CT_THREADS") == lm.CT_LOSS.stride
    assert (_const(path, "CT_TW"), _const(path, "CT_TH")) == lm.CT_TILE
    src = _src(path)
    assert "for (int j = threadIdx.x; j < a.M; j += blockDim.x)" in src          # ct_stage's strided loop
    assert "struct CtObj { int cx, cy, r; double s2; };" in src                  # 4 + 4 + 4 + pad 4 + 8 bytes
    assert re.search(r"^MAX_OBJECTS = (\d+)", _src("clean_pvnet_b200/ct_loss.py"), re.M).group(1) == str(lm.CT_LOSS.value)


def test_vote_loss_constants():
    path = lm.VOTE_LOSS.source
    assert _const(path, "VOTE_LOSS_MAX_K") == lm.VOTE_LOSS.value
    assert _const(path, "VL_THREADS") == lm.VOTE_LOSS.stride
    assert "for (int k = threadIdx.x; k < a.K; k += blockDim.x)" in _src(path)   # vote_pixel's strided loop
    assert "const size_t smem = (size_t)a.K * sizeof(double2);" in _src(path)


def test_mask_constants():
    path = lm.MASKS.source
    assert _const(path, "MASK_MAX_INSTANCES") == lm.MASKS.value
    assert _const(path, "MASK_THREADS") == lm.MASKS.stride
    src = _src(path)
    assert "struct MaskAcc { unsigned a, p, x0, x1, y0, y1; };" in src
    assert "for (int j = threadIdx.x; j < mi; j += MASK_THREADS) {" in src       # the per-instance flush
    assert "(size_t)max_m * sizeof(MaskAcc)" in src                              # the launch's dynamic shared memory


def test_decode_constants():
    path = lm.DECODE.source
    T = _const(path, "CD_T")
    assert T == lm.DECODE_TILE
    assert "constexpr int CD_N = CD_T * CD_T;" in _src(path)
    assert T * T == lm.DECODE.value
    src = _src(path)
    assert src.count("K < CD_N ? K : CD_N") == 2                                 # Lk in the launcher and the workspace
    assert "if (a.K <= a.Lk)" in src                                              # the theta bound


def test_vote_layer_constants():
    api = _src(lm.VOTE_LAYER.source)
    assert "if ((long long)d->K * ((d->hn + 511) / 512) > 65535)" in api
    assert lm.VOTE_LAYER.value == 65535
    _, path, value = lm.PRUNE_GATE
    assert "if ((long long)a.K * ((a.hn + 63) / 64) > 65535) return false;" in _src(path)
    assert value == 65535
    assert "const int k = blockIdx.y % a.K, slice = blockIdx.y / a.K;" in _src("clean_pvnet_b200/csrc/vote.cu")


def test_render_constants():
    src = _src(lm.RENDER.source)
    assert int(re.search(r"^_MAX_QUEUE = 1 << (\d+)", src, re.M).group(1)) == 26
    assert 1 << 26 == lm.RENDER.value
    assert "step = max(1, min(65535, _MAX_QUEUE // max(F, 1)))" in src
    assert "K[s:s + m] if k_stride else K" in src
    from vsd_cases import icosphere
    assert len(icosphere(lm.RENDER_SUBDIV)[1]) == lm.RENDER_FACES


# ---- the sides of each boundary ---------------------------------------------------------------------------------------

def _passes(n, stride):
    return -(-n // stride)


def test_staging_cases_straddle_the_first_pass():
    for cap in (lm.CT_LOSS, lm.VOTE_LOSS, lm.MASKS):
        lo, hi, top = cap.cases
        assert (lo, hi) == (cap.stride, cap.stride + 1) and top == cap.value, cap.op
        assert _passes(lo, cap.stride) == 1 and _passes(hi, cap.stride) == 2, cap.op
        assert _passes(top, cap.stride) == cap.value // cap.stride, cap.op
    # the stages at capacity: 24 KB of objects, 16 KB of keypoints, exactly the 48 KB a launch gets without an opt-in
    assert lm.CT_LOSS.value * lm.CT_OBJ_BYTES == 24 * 1024
    assert lm.VOTE_LOSS.value * 16 == 16 * 1024
    assert lm.MASKS.value * lm.MASK_ACC_BYTES == lm.SMEM_NO_OPT_IN
    # the mixed batch reaches both a second flush pass and the full stage in one launch
    assert max(lm.MASK_BATCH) == lm.MASKS.value and lm.MASKS.stride + 1 in lm.MASK_BATCH and 1 in lm.MASK_BATCH
    # the largest label, obj_id 30 with instance_id 2047, still fits int16
    assert lm.MAX_OBJ_ID * 1000 + lm.MASKS.value - 1 <= lm.INT16_MAX


def test_ct_crowded_tile_holds_every_object():
    tw, th = lm.CT_TILE
    assert tw * th >= lm.CT_LOSS.stride * 2               # a tile has room for 512 distinct centres
    assert lm.CT_SHAPE["H"] >= th and lm.CT_SHAPE["W"] >= tw


def test_decode_cases_straddle_the_list_cap():
    H, W = lm.DECODE_SHAPE["H"], lm.DECODE_SHAPE["W"]
    k1024, k1025, k4096, kfull = lm.DECODE.cases
    N = lm.DECODE.value

    def theta_bound(K):                                   # ct_decode_select_kernel: theta only when K <= Lk
        return K <= min(K, N)
    assert k1024 == N and theta_bound(k1024)
    assert k1025 == N + 1 and not theta_bound(k1025)
    assert k4096 > N and not theta_bound(k4096)
    assert kfull == H * W == 13312 and not theta_bound(kfull)
    # every case is accepted (K <= H*W, C*K < 2^24) and ranked by a loop of at most H*W steps
    for K in lm.DECODE.cases:
        for C in lm.DECODE_SHAPE["C"]:
            assert K <= H * W and C * K < 1 << 24
    # a 32x32 tile holds N keys, so a saturated tile alone fills the top K at K = N
    assert lm.DECODE_TILE ** 2 == N


def test_vote_layer_cases_straddle_the_prune_gate_and_the_abi_limit():
    hn = lm.VOTE_LAYER_HN
    k_pruned, k_unpruned, k_max = lm.VOTE_LAYER.cases
    B = lm.VOTE_LAYER_SHAPE["B"]
    assert prune_applies(0.99, hn, B[k_pruned], k_pruned)
    assert not prune_applies(0.99, hn, B[k_unpruned], k_unpruned)
    assert k_pruned * -(-hn // 64) <= 65535 < k_unpruned * -(-hn // 64)
    # the ABI's limit: K = 16383 is its largest K at hn = 2048
    assert k_max * -(-hn // 512) <= lm.VOTE_LAYER.value < (k_max + 1) * -(-hn // 512)
    assert not prune_applies(0.99, hn, B[k_max], k_max)
    # the K = 1 calls the big ones are compared with are accepted and never pruned
    assert not prune_applies(0.99, hn, 2, 1)
    # the distribution's hypothesis count at K = 16383
    assert lm.DIST_ROUND_HN * -(-hn // lm.DIST_ROUND_HN) == hn
    for K in lm.VOTE_LAYER.cases:
        ks = lm.vote_keypoints(K)
        assert 12 <= len(ks) <= 20 and ks[0] == 0 and ks[-1] == K - 1 and len(set(ks)) == len(ks)


def test_render_poses_fall_in_two_launches():
    step = lm.render_step(lm.RENDER_FACES)
    assert step == 3276
    n = lm.RENDER.cases[0]
    assert step < n < 2 * step
    launch = [p // step for p in lm.RENDER_POSES]
    assert launch == [0, 0, 1, 1] and lm.RENDER_POSES[1] + 1 == lm.RENDER_POSES[2] == step
    assert lm.RENDER_POSES[-1] == n - 1


# ---- budgets ----------------------------------------------------------------------------------------------------------

def test_device_bytes_fit_the_budget():
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    lib = _lib.load()
    sizes = {}
    for M in lm.CT_LOSS.cases:
        for C in lm.CT_SHAPE["C"]:
            sizes[f"ct M={M} C={C}"] = lm.ct_bytes(M, C)
    for K in lm.VOTE_LOSS.cases:
        sizes[f"vote_loss K={K}"] = lm.vote_loss_bytes(K)
    for m in lm.MASKS.cases:
        sizes[f"masks {m}"] = lm.mask_bytes([m])
    sizes["masks batch"] = lm.mask_bytes(lm.MASK_BATCH)
    for K in lm.DECODE.cases:
        for C in lm.DECODE_SHAPE["C"]:
            sizes[f"decode K={K} C={C}"] = lm.decode_bytes(K, C)
    for K in lm.VOTE_LAYER.cases:
        assert lm.vote_workspace_bytes(K) > 0, K
        sizes[f"vote layer K={K}"] = lm.vote_layer_bytes(K)
    assert lib.pvb_render_depth_workspace_bytes(lm.render_step(lm.RENDER_FACES), lm.RENDER_FACES) <= lm.render_bytes()
    sizes["render"] = lm.render_bytes()
    for name, n in sizes.items():
        print(f"{name}: {n / 2 ** 20:.0f} MiB")
        assert 0 < n <= lm.DEVICE_BUDGET, name


def _timed(f, *args, **kw):
    t = time.perf_counter()
    out = f(*args, **kw)
    return out, time.perf_counter() - t


def test_restatements_are_cheap_at_the_largest_cases():
    from ct_target_cases import restate_batch
    from vote_target_cases import restate_vertex
    from tless_mask_cases import compose_restated
    import ct_decode_cases as dc
    rng = np.random.default_rng(0)
    times = {}
    # ct: four images of 1024 objects each, thirty classes
    B, H, W, M = lm.CT_SHAPE["B"], lm.CT_SHAPE["H"], lm.CT_SHAPE["W"], lm.CT_LOSS.value
    ind = rng.integers(0, H * W, (B, M))
    _, times["ct"] = _timed(restate_batch, ind, rng.integers(0, 30, (B, M)).astype(np.int32),
                            rng.integers(0, 30, (B, M)), np.ones((B, M), np.float32), 30, H, W)
    # vote loss: one image, 1024 keypoints, a third of it foreground
    H, W, K = lm.VOTE_LOSS_SHAPE["H"], lm.VOTE_LOSS_SHAPE["W"], lm.VOTE_LOSS.value
    _, times["vote_loss"] = _timed(restate_vertex, (rng.random((H, W)) < 0.35).astype(np.uint8),
                                   rng.uniform(-20, 100, (K, 2)))
    # masks: 2048 instances on one image
    H, W = lm.MASK_SHAPE["H"], lm.MASK_SHAPE["W"]
    depth = np.where(rng.random((lm.MASKS.value, H, W)) < 0.05, 800.0, 0.0).astype(np.float32)
    _, times["masks"] = _timed(compose_restated, depth, np.full(lm.MASKS.value, 30))
    # decode: the stable-sort restatement at K = H*W (on the CPU here; the GPU test runs it on CUDA torch)
    H, W = lm.DECODE_SHAPE["H"], lm.DECODE_SHAPE["W"]
    lg = torch.from_numpy(dc.blobs(rng, 2, 1, H, W, noise=0.3))
    _, times["decode"] = _timed(dc.restate_decode_ordered, lg, torch.zeros(2, 2, H, W), H * W)
    for name, t in times.items():
        print(f"{name}: {t:.2f} s")
        assert t <= lm.RESTATE_SECONDS, name


def test_oracles_are_cheap_at_the_largest_cases(oracle):
    """The vote layer's CPU oracle on one keypoint of a two-image call at hn = 2048, and the render oracle on one
    icosphere(5) pose: the GPU test calls each a few dozen and two times."""
    import render_oracle
    from vsd_cases import K_SMALL, icosphere, poses
    B, H, W, hn = 2, lm.VOTE_LAYER_SHAPE["H"], lm.VOTE_LAYER_SHAPE["W"], lm.VOTE_LAYER_HN
    rng = np.random.default_rng(1)
    v = rng.normal(size=(B, H, W, 1, 2)).astype(np.float32)
    idxs = rng.integers(0, H * W, (B, hn, 1, 2)).astype(np.int32)
    _, t = _timed(oracle.ransac_voting_layer_v3, np.ones((B, H, W), np.int64), v, hn, inlier_thresh=0.99, idxs=idxs,
                  debug=True)
    assert t <= lm.RESTATE_SECONDS / 10, t
    render_oracle.build()
    pts, faces = icosphere(lm.RENDER_SUBDIV)
    K = K_SMALL.copy()
    K[0, 2], K[1, 2] = lm.RENDER_SIZE[0] / 2, lm.RENDER_SIZE[1] / 2
    _, t = _timed(render_oracle.render_depth, pts, faces, poses(1, seed=0)[0], K, lm.RENDER_SIZE)
    assert t <= lm.RESTATE_SECONDS, t
