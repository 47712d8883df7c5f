"""A restatement of the CenterNet detector's decode (Network.decode_detection: torch.sigmoid, decode_ct_hm and
clip_to_image) in plain torch ops, and the seeded cases the tests and tests/golden/make_golden_ct_decode.py run it on.
The restatement runs on CPU or CUDA torch; on CUDA it is the yardstick the fused decode is pinned to, ties included."""
import numpy as np
import torch
import torch.nn.functional as F

from ct_target_cases import restate_ct_hm

# the detector's output sizes: (H, W) at its test input 736x544 and at its training input 512x416
TEST_HW, TRAIN_HW = (136, 184), (104, 128)


def _peaks(ct_hm):
    """sigmoid and the 3x3 peak test: max_pool2d (stride 1, pad 1); heat where the pool equals it, else heat * 0."""
    heat = torch.sigmoid(ct_hm)
    hmax = F.max_pool2d(heat, (3, 3), stride=1, padding=1)
    return heat * (hmax == heat).float()


def _detections(score, cls, ind, wh, K, clip, h, w):
    """The rows of the K winners: ct (xs, ys) and detection (box, score, class), then clip_to_image to (h, w)."""
    B, _, H, W = wh.shape
    ys = (ind / W).int().float()
    xs = (ind % W).int().float()
    sz = wh.permute(0, 2, 3, 1).reshape(B, H * W, 2).gather(1, ind[:, :, None].expand(B, K, 2))
    half_w, half_h = sz[..., 0] / 2, sz[..., 1] / 2
    boxes = torch.stack([xs - half_w, ys - half_h, xs + half_w, ys + half_h], dim=2)
    if clip:
        boxes[..., :2] = torch.clamp(boxes[..., :2], min=0)
        boxes[..., 2] = torch.clamp(boxes[..., 2], max=(W if w is None else w) - 1)
        boxes[..., 3] = torch.clamp(boxes[..., 3], max=(H if h is None else h) - 1)
    ct = torch.stack([xs, ys], dim=2)
    det = torch.cat([boxes, score[..., None], cls.float()[..., None]], dim=2)
    return ct, det


def restate_decode(ct_hm, wh, K=100, clip=True, h=None, w=None):
    """Network.decode_detection(output, h, w) of output = {'ct_hm': ct_hm, 'wh': wh} on ct_hm's device, step by step:
    sigmoid; the 3x3 peak test; topk of K per class over the flattened map; topk of K over the C*K winners;
    ys = (ind / W).int().float(), xs = ind % W, class = (j / K).int(); wh gathered at the winner's pixel; the box
    xs -+ w/2, ys -+ h/2; then clip_to_image to (h, w) (default: the map's own size).  Returns (ct [B,K,2], detection
    [B,K,6]).  Any strides are accepted (the reference's .view needs a contiguous map; reshape gives it the same
    values).  Equal values come out in whatever order torch.topk leaves them."""
    B, C, H, W = ct_hm.shape
    heat = _peaks(ct_hm)
    s1, i1 = torch.topk(heat.reshape(B, C, H * W), K)
    i1 = i1 % (H * W)
    score, j = torch.topk(s1.reshape(B, C * K), K)
    cls = (j / K).int()
    ind = i1.reshape(B, C * K).gather(1, j)
    return _detections(score, cls, ind, wh, K, clip, h, w)


def restate_decode_ordered(ct_hm, wh, K=100, clip=True, h=None, w=None):
    """restate_decode with the two topk replaced by one stable sort of each image's C*H*W values, descending: the same
    rows, with equal values ordered by class and then by pixel index (NaN first, as topk ranks it)."""
    B, C, H, W = ct_hm.shape
    heat = _peaks(ct_hm).reshape(B, C * H * W)
    score, j = torch.sort(heat, dim=1, descending=True, stable=True)
    score, j = score[:, :K], j[:, :K]
    return _detections(score, (j // (H * W)).int(), j % (H * W), wh, K, clip, h, w)


# ---- seeded cases: (name, ct_hm logits float32 [B,C,H,W], wh float32 [B,2,H,W], K) on the CPU --------------------------

def _logit(p):
    p = np.clip(np.asarray(p, np.float64), 1e-7, 1 - 1e-7)
    return np.log(p / (1 - p)).astype(np.float32)


def _wh(rng, B, H, W, top=60.0):
    return rng.uniform(0.0, top, (B, 2, H, W)).astype(np.float32)


def blobs(rng, B, C, H, W, objects=6, noise=0.0):
    """Gaussian blobs (the datasets' draw_umich_gaussian, ct_target_cases) per class, plus uniform noise, as logits
    (probabilities above 1 - 1e-7 saturate, so strong noise on a blob's top makes ties)."""
    hm = np.zeros((B, C, H, W), np.float32)
    for b in range(B):
        M = objects * C
        ind = rng.integers(0, H * W, M)
        rad = rng.integers(0, max(1, min(H, W) // 4), M)
        cls = rng.integers(0, C, M)
        hm[b] = restate_ct_hm(ind, rad, cls, np.ones(M, np.float32), C, H, W)
    p = 0.02 + 0.96 * hm + noise * rng.uniform(0, 1, hm.shape)
    return _logit(p)


def tie_free(rng, B, C, H, W, K):
    """Blobs plus noise where neither top-K meets a tie (each class's K + 1 largest values are distinct, and so are the
    K + 1 largest of the classes' winners), so the CPU torch topk (whose tie order is not CUDA's) picks and orders every
    row the same way."""
    def distinct(v):
        return bool((v[:-1] > v[1:]).all())
    for _ in range(100):
        lg = blobs(rng, B, C, H, W) + rng.uniform(-2.0, 0.0, (B, C, H, W)).astype(np.float32)
        heat = torch.sigmoid(torch.from_numpy(lg))
        heat = (heat * (F.max_pool2d(heat, 3, stride=1, padding=1) == heat).float()).reshape(B, C, H * W)
        top = torch.sort(heat, dim=2, descending=True).values[..., :K + 1]
        second = torch.sort(top[..., :K].reshape(B, C * K), dim=1, descending=True).values[:, :K + 1]
        if all(distinct(t) for t in top.reshape(B * C, -1)) and all(distinct(t) for t in second):
            return lg
    raise RuntimeError("no tie-free heatmap found")


def cases(seed=20261017):
    """Every semantic corner the decode has, ties and NaN included: [(name, logits, wh, K)]."""
    rng = np.random.default_rng(seed)
    out = []
    H, W = TEST_HW
    out.append(("blobs_noise_c1", blobs(rng, 2, 1, H, W, noise=0.3), _wh(rng, 2, H, W), 100))
    # few peaks: clean blobs, so every class has fewer than K peaks and the zero tail fills the rows
    out.append(("few_peaks_c30", blobs(rng, 2, 30, *TRAIN_HW, objects=1), _wh(rng, 2, *TRAIN_HW), 100))
    # saturated logits: sigmoid gives exact 0 and 1, plateaus of equal values, all of them kept
    lg = rng.choice(np.array([-np.inf, -30, 30, np.inf, 0.0], np.float32), (2, 3, 24, 20))
    lg[:, :, 5:9, 5:9] = 30.0
    out.append(("saturated", lg, _wh(rng, 2, 24, 20), 50))
    # two distinct logits with one sigmoid: both survive the peak test
    lg = np.full((1, 2, 9, 11), -5.0, np.float32)
    lg[0, 0, 2, 2], lg[0, 0, 2, 3] = 20.0, 21.0        # sigmoid rounds both to exactly 1
    lg[0, 1, 6, 8] = 20.5
    out.append(("sigmoid_ties", lg, _wh(rng, 1, 9, 11), 12))
    # the same scores in two classes
    lg = blobs(rng, 2, 4, 40, 36, noise=0.2)
    lg[:, 2] = lg[:, 0]
    lg[:, 3] = lg[:, 1]
    out.append(("same_score_two_classes", lg, _wh(rng, 2, 40, 36), 100))
    # NaN logits: the NaN pixel stays NaN and ranks first, its neighbours become 0
    lg = blobs(rng, 2, 3, 30, 26, noise=0.3)
    lg[0, 0, 10, 10] = np.nan
    lg[0, 1, 0, 0] = np.nan
    lg[1, 2, 29, 25] = np.nan
    lg[1, 2, 15, 3] = np.nan
    out.append(("nan", lg, _wh(rng, 2, 30, 26), 40))
    # peaks on the borders and at the corners
    lg = np.full((1, 1, 17, 23), -4.0, np.float32)
    for (y, x, v) in [(0, 0, 3.0), (0, 22, 2.5), (16, 0, 2.0), (16, 22, 1.5), (0, 11, 1.0), (8, 0, 0.5), (16, 9, 0.25),
                      (7, 22, 0.125)]:
        lg[0, 0, y, x] = v
    out.append(("borders", lg, _wh(rng, 1, 17, 23), 20))
    # K = H*W and odd sizes
    out.append(("k_full_7x5", blobs(rng, 2, 2, 5, 7, noise=0.5), _wh(rng, 2, 5, 7), 35))
    out.append(("odd_7x5", blobs(rng, 3, 3, 5, 7, noise=0.2), _wh(rng, 3, 5, 7), 8))
    # the detector's shapes, C in {1, 30}
    for C in (1, 30):
        for hw in (TEST_HW, TRAIN_HW):
            out.append((f"detector_c{C}_{hw[0]}x{hw[1]}", blobs(rng, 2, C, *hw, noise=0.3), _wh(rng, 2, *hw), 100))
    # wh large enough that clipping bites on every side
    out.append(("clip", blobs(rng, 1, 2, 30, 40, noise=0.3), rng.uniform(0, 200, (1, 2, 30, 40)).astype(np.float32), 60))
    return out


def golden_cases(seed=20261018):
    """Tie-free cases for the CPU-made fixture: [(name, logits, wh, K)]."""
    rng = np.random.default_rng(seed)
    return [("tiefree_c1_test", tie_free(rng, 1, 1, *TEST_HW, 100), _wh(rng, 1, *TEST_HW, 400.0), 100),
            ("tiefree_c2_train", tie_free(rng, 1, 2, *TRAIN_HW, 100), _wh(rng, 1, *TRAIN_HW, 400.0), 100),
            ("tiefree_small", tie_free(rng, 2, 2, 12, 15, 5), rng.uniform(0, 40, (2, 2, 12, 15)).astype(np.float32), 5)]


# detection_boxes' reference frame: the detector's test input and the meta of a 720x540 T-LESS image
BOX_INPUT_SIZE = (736, 544)
BOX_CENTER = (360.0, 270.0)
BOX_SCALE = (720.0, 720.0)
