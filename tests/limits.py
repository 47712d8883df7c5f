"""The capacity each batched op's C ABI accepts, and the case sizes tests/test_gpu_limits.py runs on both sides of it.

Every capacity is the size of a shared-memory stage, a list or a launch split.  Below it a loop runs once or a branch
takes the path every other test reaches; at it the loop runs several times or the branch switches.  Each row names the
constant and the file it is stated in, its value, the thread stride of the loop that walks it (None where there is no
loop), and the cases.  tests/test_limits_host.py parses every constant out of its source and checks it against this
table, and checks that each case lies on the side of its boundary the table says, so a changed capacity fails there
until the cases follow it.  It also checks each case's device bytes (the shapes below, worked out by hand) and the
cost of its CPU restatement against a budget."""
import math
from collections import namedtuple

Capacity = namedtuple("Capacity", "op constant source value stride cases")

GB = 1 << 30
DEVICE_BUDGET = 2 * GB           # peak device memory of any one case: the GPUs are shared
RESTATE_SECONDS = 5.0            # each case's CPU restatement

# ---- ct_focal_loss / CenterNet target (csrc/ct_loss.cu) --------------------------------------------------------------
# ct_stage stages the objects of one (tile, class, image) 256 threads at a time, 24 bytes each.  Every image holds M
# objects; with C = 1 they are crowded into one 32x16 tile, whose staged list then holds all M.
CT_LOSS = Capacity("ct_focal_loss", "CT_MAX_M", "clean_pvnet_b200/csrc/ct_loss.cu", 1024, 256, (256, 257, 1024))
CT_SHAPE = dict(B=4, H=104, W=128, C=(30, 1))
CT_OBJ_BYTES = 24                # sizeof(CtObj)
CT_TILE = (32, 16)               # CT_TW x CT_TH

# ---- vote_loss / vote target (csrc/loss.cu) --------------------------------------------------------------------------
# vote_pixel stages the image's keypoints 256 threads at a time, as double2.
VOTE_LOSS = Capacity("vote_loss", "VOTE_LOSS_MAX_K", "clean_pvnet_b200/csrc/loss.cu", 1024, 256, (256, 257, 1024))
VOTE_LOSS_SHAPE = dict(B=2, H=64, W=80)

# ---- instance_masks_* compose (csrc/render.cu) -----------------------------------------------------------------------
# mask_compose_kernel keeps max_m * 24 bytes of per-instance sums in dynamic shared memory and flushes them 256 threads
# at a time.  Cases: one image of each size, then one batch of three images.
MASKS = Capacity("instance_masks", "MASK_MAX_INSTANCES", "clean_pvnet_b200/csrc/render.cu", 2048, 256, (256, 257, 2048))
MASK_BATCH = (2048, 1, 257)
MASK_SHAPE = dict(H=61, W=83, slots=40)
MASK_ACC_BYTES = 24              # sizeof(MaskAcc)
SMEM_NO_OPT_IN = 48 * 1024       # dynamic shared memory a launch gets without cudaFuncAttributeMaxDynamicSharedMemorySize
INT16_MAX = 32767
MAX_OBJ_ID = 30                  # T-LESS's obj_ids run 1..30

# ---- decode_detections (csrc/ct_decode.cu) ---------------------------------------------------------------------------
# Each 32x32 tile lists its Lk = min(K, CD_N) largest keys; the theta bound needs K <= Lk.  The last case, K = H*W, selects
# every key of the training map; its O(K^2) ranking runs in one CTA per image, so K stays far below the ABI's 2^24.
DECODE = Capacity("decode_detections", "CD_N", "clean_pvnet_b200/csrc/ct_decode.cu", 1024, None,
                  (1024, 1025, 4096, 104 * 128))
DECODE_SHAPE = dict(B=2, H=104, W=128, C=(3, 1))    # C = 1 only for K = H*W
DECODE_TILE = 32

# ---- ransac_voting_layer_v3 / estimate_voting_distribution_with_mean (csrc/api.cu, prune.cu, vote.cu) -----------------
# The ABI accepts K * ceil(hn / 512) <= 65535; the pruned vote also needs K * ceil(hn / 64) <= 65535.
VOTE_LAYER = Capacity("ransac_voting_layer_v3", "K*ceil(hn/512) <= 65535", "clean_pvnet_b200/csrc/api.cu", 65535, None,
                      (2047, 2048, 16383))
VOTE_LAYER_HN = 2048
VOTE_LAYER_SHAPE = dict(H=24, W=32, B={2047: 2, 2048: 2, 16383: 1})
PRUNE_GATE = ("K*ceil(hn/64) <= 65535", "clean_pvnet_b200/csrc/prune.cu", 65535)
DIST_ROUND_HN = 256              # estimate_voting_distribution_with_mean at K = 16383: 8 rounds of 256 = VOTE_LAYER_HN


def vote_keypoints(K):
    """The keypoints whose results the GPU test checks one by one: the first and last two, both sides of each multiple
    of K / 16, and the middle."""
    ks = {0, 1, K // 2, K - 2, K - 1}
    for i in range(1, 6):
        j = i * K // 6
        ks |= {j - 1, j}
    return sorted(k for k in ks if 0 <= k < K)


# ---- render_depth_batch (render.py) ----------------------------------------------------------------------------------
# _render splits the poses into launches of min(65535, _MAX_QUEUE // F) and slices a per-pose K with them.
RENDER = Capacity("render_depth_batch", "_MAX_QUEUE", "clean_pvnet_b200/render.py", 1 << 26, None, (3300,))
RENDER_SUBDIV = 5                # icosphere(5): 20 * 4^5 = 20480 faces
RENDER_FACES = 20 * 4 ** RENDER_SUBDIV
RENDER_SIZE = (64, 48)           # (width, height)
RENDER_POSES = (0, 3275, 3276, 3299)


def render_step(F, queue=RENDER.value):
    return max(1, min(65535, queue // max(F, 1)))


# ---- device bytes, worked out from the shapes -------------------------------------------------------------------------
def ct_bytes(M, C):
    B, H, W = CT_SHAPE["B"], CT_SHAPE["H"], CT_SHAPE["W"]
    n = B * C * H * W * 4
    # logits, two leaves and their gradients, the dense target and autograd's saved intermediates (under a dozen maps)
    return 16 * n + 4 * B * M * 8


def vote_loss_bytes(K):
    B, H, W = VOTE_LOSS_SHAPE["B"], VOTE_LOSS_SHAPE["H"], VOTE_LOSS_SHAPE["W"]
    n = B * 2 * K * H * W * 4
    return 16 * n


def mask_bytes(counts):
    H, W, S = MASK_SHAPE["H"], MASK_SHAPE["W"], MASK_SHAPE["slots"]
    n = sum(counts)
    return S * H * W * 4 + len(counts) * H * W * 2 + n * (8 + 8 + 16 + 2 * 4 + MASK_ACC_BYTES) + 4096


def decode_bytes(K, C):
    B, H, W = DECODE_SHAPE["B"], DECODE_SHAPE["H"], DECODE_SHAPE["W"]
    tiles = math.ceil(H / DECODE_TILE) * math.ceil(W / DECODE_TILE)
    lists = B * C * tiles * min(K, DECODE.value) * 8
    maps = (C + 2) * B * H * W * 4
    # the stable-sort restatement keeps a few copies of the C*H*W values and their int64 indices
    return lists + B * K * 8 + B * K * 8 * 4 + maps + 8 * B * C * H * W * 12


def vote_workspace_bytes(K):
    """pvb_workspace_bytes of the case's calls (the larger of the two selection modes; host code, no device needed)."""
    import torch
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    B, H, W = VOTE_LAYER_SHAPE["B"][K], VOTE_LAYER_SHAPE["H"], VOTE_LAYER_SHAPE["W"]
    m, v = torch.ones(B, H, W, dtype=torch.uint8), torch.zeros(B, H, W, K, 2)
    return max(_lib.load().pvb_workspace_bytes(rv._make_desc(m, v, VOTE_LAYER_HN, 0.99, 5, 30000, sel, 0, 0, None))
               for sel in (_lib.PVB_SELECT_BYTE, _lib.PVB_SELECT_EQ1))


def vote_layer_bytes(K):
    """The workspace, which the operator allocates 1.25 times over, the field, the sample pairs and the outputs."""
    workspace = vote_workspace_bytes(K)
    B, H, W = VOTE_LAYER_SHAPE["B"][K], VOTE_LAYER_SHAPE["H"], VOTE_LAYER_SHAPE["W"]
    vertex = B * H * W * K * 2 * 4
    idxs = B * VOTE_LAYER_HN * K * 2 * 4
    return int(workspace * 1.25) + 256 + 2 * vertex + idxs + B * K * 2 * 4 * 4


def render_bytes(n=RENDER.cases[0], F=RENDER_FACES):
    W, H = RENDER_SIZE
    V = 2 + 10 * 4 ** RENDER_SUBDIV
    return n * H * W * 4 + 256 + render_step(F) * F * 4 + n * 9 * 8 + n * 12 * 8 + V * 12 + F * 12
