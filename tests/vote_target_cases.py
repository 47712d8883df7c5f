"""The inputs of tests/golden/vote_target.npz and a numpy restatement of compute_vertex
(lib/utils/pvnet/pvnet_data_utils.py:30-44), shared by the fixture's generator and the tests."""
import numpy as np

# (K, H, W) of each case; every case holds three images
SHAPES = [(1, 9, 13), (9, 12, 16), (17, 20, 24)]


def restate_vertex(mask, kpt_2d):
    """compute_vertex(mask, kpt_2d).transpose(2, 0, 1) in plain numpy: mask [H,W], kpt_2d [K,2] -> float32 [2K,H,W].
    The norm is sqrt(dx*dx + dy*dy) (what np.linalg.norm computes; np.hypot rounds differently)."""
    kpt = np.asarray(kpt_2d, np.float64)
    ys, xs = np.nonzero(np.asarray(mask) == 1)
    dx = kpt[None, :, 0] - xs[:, None].astype(np.float64)
    dy = kpt[None, :, 1] - ys[:, None].astype(np.float64)
    n = np.sqrt(dx * dx + dy * dy)
    n = np.where(n < 1e-3, n + 1e-3, n)
    out = np.zeros((2 * kpt.shape[0],) + np.asarray(mask).shape, np.float32)
    out[0::2, ys, xs] = (dx / n).T
    out[1::2, ys, xs] = (dy / n).T
    return out


def case_inputs(seed=20261016):
    """[(mask uint8 [3,H,W], kpt float64 [3,K,2])] for SHAPES.  The masks hold 0, 1, 2 and 255; the keypoints include
    points exactly on a pixel (n = 0 -> 1e-3, a zero vector), within 1e-3 of a pixel, at +-1e6 px and at negative
    coordinates, besides ordinary ones."""
    rng = np.random.default_rng(seed)
    out = []
    for K, H, W in SHAPES:
        mask = rng.choice(np.array([0, 1, 1, 1, 2, 255], np.uint8), size=(3, H, W))
        kpt = np.stack([rng.uniform(-5, W + 5, (3, K)), rng.uniform(-5, H + 5, (3, K))], -1)
        special = [
            (3.0, 4.0),                          # on a pixel
            (5.0 + 3e-4, 2.0 - 4e-4),            # within 1e-3 of one
            (1e6, -1e6), (-1e6, 1e6),
            (-2.5, -7.25),
            (7.0, 1.0 + 1e-9),
            (2.0 - 6e-4, 6.0),
        ]
        for i in range(3):
            for j in range(K):
                if (i + j) % 2 == 0 or K == 1:
                    kpt[i, j] = special[(i * K + j) % len(special)]
        # make the on-pixel keypoints' pixels foreground, so the zero vector is exercised
        for i in range(3):
            for j in range(K):
                x, y = kpt[i, j]
                if x == int(x) and y == int(y) and 0 <= x < W and 0 <= y < H:
                    mask[i, int(y), int(x)] = 1
        out.append((mask, kpt))
    return out
