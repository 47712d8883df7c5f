"""The inputs of tests/golden/ct_target.npz and a numpy restatement of the CenterNet datasets' heatmap target
(data_utils.gaussian2D + draw_umich_gaussian, lib/utils/data_utils.py:36-64, as lib/datasets/tless*/ct.py calls them),
shared by the fixture's generator and the tests."""
import math

import numpy as np

# (B, C, H, W) of each case; case 0 is hand-made, cases 1 and 2 are the detector's training and validation outputs
SHAPES = [(4, 3, 20, 24), (2, 30, 104, 128), (1, 30, 136, 184)]


def restate_ct_hm(ct_ind, ct_radius, ct_cls, ct_01, C, H, W):
    """One image's ct_hm in plain numpy: the objects are [M] arrays -> float32 [C,H,W].  Per pixel of an object's window
    (clipped to the image), g = exp(-(dx*dx / s2 + dy*dy / s2) / 2) in fp64 with s2 = ((2r + 1) / 6)^2, g < 2^-52 -> 0,
    and the heatmap keeps float32(max(old, g)).  Objects with ct_01 != 1, a class outside [0, C) or a centre off the
    image draw nothing."""
    out = np.zeros((C, H, W), np.float32)
    for ind, r, c, v in zip(np.asarray(ct_ind).tolist(), np.asarray(ct_radius).tolist(), np.asarray(ct_cls).tolist(),
                            np.asarray(ct_01).tolist()):
        if v != 1 or not 0 <= c < C or r < 0 or not 0 <= ind < H * W:
            continue
        cy, cx = divmod(int(ind), W)
        x0, x1, y0, y1 = max(0, cx - r), min(W, cx + r + 1), max(0, cy - r), min(H, cy + r + 1)
        dx = np.arange(x0, x1, dtype=np.float64) - cx
        dy = np.arange(y0, y1, dtype=np.float64) - cy
        sigma = (2 * r + 1) / 6
        s2 = sigma * sigma
        g = np.exp(-((dx * dx / s2)[None, :] + (dy * dy / s2)[:, None]) / 2)
        g[g < np.finfo(np.float64).eps] = 0
        out[c, y0:y1, x0:x1] = np.maximum(out[c, y0:y1, x0:x1], g)
    return out


def centre(box):
    """prepare_detection's centre of an (x_min, y_min, x_max, y_max) box: the float32 midpoint rounded half to even."""
    x0, y0, x1, y1 = box
    ct = np.round(np.array([(x0 + x1) / 2, (y0 + y1) / 2], dtype=np.float32)).astype(np.int32)
    return int(ct[0]), int(ct[1])


def _edge_images(W, H):
    """Case 0's four images as [(box, cls)]: radius-0 boxes; centres on the four borders and the corners (given as
    ("ct", cx, cy, r), since a box clipped to the image has a small extent across a border centre); same-class
    overlapping windows and different classes at one centre; half-pixel centres and float boxes whose height lies just
    above an integer (float32 rounds it onto the integer); and an image with no objects."""
    borders = [((0, 0, 1, 1), 0), ((0, 3, 0.9, 3.8), 1), ((10, 10, 11, 11), 2),     # r = 0 (ceil sizes 1)
               (("ct", 0, 10, 5), 0), (("ct", W - 1, 7, 6), 1), (("ct", 12, 0, 4), 2), (("ct", 8, H - 1, 3), 0),
               (("ct", 0, 0, 7), 2), (("ct", W - 1, 0, 2), 1), (("ct", 0, H - 1, 9), 1), (("ct", W - 1, H - 1, 25), 2),
               (("ct", 15, 15, 0), 0)]
    overlap = [((2, 2, 14, 12), 0), ((6, 5, 18, 15), 0), ((8, 7, 12, 9), 0),
               ((5, 5, 15, 15), 1), ((7, 7, 13, 13), 2), ((3, 3, 17, 17), 1)]                  # one centre, 3 boxes
    halves = [((2, 2, 7, 9), 0), ((4, 3, 11, 12), 1), ((13, 2.5, 18, 7.5), 2), ((1.25, 11, 8.75, 17), 0),
              ((14, 10, 21.5, 10 + 7 + 1e-7), 1), ((3, 1, 9.0000001, 8), 2), ((16, 12.2, 22, 19.2000001), 0)]
    return [borders, overlap, halves, []]


def case_images(seed=20261017):
    """[(B, C, H, W, images)] for SHAPES, each image a list of (box, cls) as prepare_detection receives them (boxes
    already clipped to the output, never empty)."""
    rng = np.random.default_rng(seed)
    out = [(4, 3, 20, 24, _edge_images(24, 20))]
    for B, C, H, W in SHAPES[1:]:
        images = []
        for b in range(B):
            objs = []
            for _ in range(int(rng.integers(12, 21))):
                w, h = rng.uniform(1, 0.5 * W), rng.uniform(1, 0.5 * H)
                x0, y0 = rng.uniform(-0.1 * W, W - 2), rng.uniform(-0.1 * H, H - 2)
                box = [max(0.0, x0), max(0.0, y0), min(W - 1.0, x0 + w), min(H - 1.0, y0 + h)]
                if b % 2 == 0:                                  # cv2.boundingRect's integer boxes
                    box = [float(math.floor(v)) for v in box]
                if box[2] - box[0] <= 1 or box[3] - box[1] <= 1:
                    continue
                objs.append((tuple(box), int(rng.integers(0, C))))
            objs.append((objs[0][0], (objs[0][1] + 1) % C))     # a second class at one centre
            images.append(objs)
        out.append((B, C, H, W, images))
    return out


def pack(images, W, radius_fn):
    """The collator's padded [B,M] arrays of a batch of images: ct_ind int64, ct_radius int32 (radius_fn(h, w) of the
    box's float64 height and width), ct_cls int64, ct_01 float32, and wh float64 [B,M,2] (w, h; NaN for an object
    given as ("ct", cx, cy, r))."""
    B, M = len(images), max([len(o) for o in images] + [0])
    ind, rad, cls = np.zeros((B, M), np.int64), np.zeros((B, M), np.int32), np.zeros((B, M), np.int64)
    c01, wh = np.zeros((B, M), np.float32), np.zeros((B, M, 2), np.float64)
    for b, objs in enumerate(images):
        for j, (box, c) in enumerate(objs):
            if box[0] == "ct":
                _, cx, cy, r = box
                w = h = np.nan
            else:
                cx, cy = centre(box)
                h, w = box[3] - box[1], box[2] - box[0]
                r = radius_fn(h, w)
            ind[b, j], rad[b, j], cls[b, j], c01[b, j] = cy * W + cx, r, c, 1
            wh[b, j] = (w, h)
    return ind, rad, cls, c01, wh


def restate_batch(ind, rad, cls, c01, C, H, W):
    return np.stack([restate_ct_hm(ind[b], rad[b], cls[b], c01[b], C, H, W) for b in range(ind.shape[0])]) \
        if ind.shape[0] else np.zeros((0, C, H, W), np.float32)
