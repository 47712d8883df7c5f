"""Numpy restatement of T-LESS's PVNet crop (DESIGN.md 8g): the crop matrix of data_utils.get_affine_transform
(lib/utils/data_utils.py:123-156) with cv2.getAffineTransform's 6x6 LU, cv2.warpAffine(INTER_LINEAR)'s fixed-point
bilinear, magnify_box and the normalisation of tless_test_utils.pvnet_transform (lib/utils/tless/tless_test_utils.py:
57-77), and the un-crop of the evaluator (lib/evaluators/tless_test/pvnet.py:229-239).  Every step is written in the
order and precision the device kernels (csrc/crop.cu) use, so the tests can pin the kernels to this file and this file to
cv2 and to the reference's own outputs (tests/golden/tless_crop.npz).  Case generators for both live here too."""
import numpy as np

MEAN = np.array([0.40789654, 0.44719302, 0.47026115], np.float32)     # lib/utils/tless/tless_config.py
STD = np.array([0.28863828, 0.27408164, 0.27809835], np.float32)
CONFIGS = {"256": ((256, 256), 2.4, 1.2), "128": ((128, 128), 1.2, 1.1)}   # (input_size, scale_ratio, box_ratio)
LU_EPS = np.finfo(np.float64).eps * 100                                    # hal::LU64f's pivot threshold
f32 = np.float32


def _fma(a, b, c):
    """a * b + c rounded once (what OpenBLAS's dgemm kernel does in np.dot on x86-64)."""
    from fractions import Fraction
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def crop_points(center, scale, out_w, out_h):
    """src, dst float32 [3,2] of get_affine_transform(center, scale, 0, [out_w, out_h]) under numpy 2's promotions:
    center is used in float64 (a float32 centre is exact in it), scale is rounded to float32, and center + src_dir is
    formed in float64 before it is stored into the float32 array."""
    cx, cy = float(center[0]), float(center[1])
    v = float(f32(f32(scale) * f32(-0.5)))                  # src_w * -0.5, float32 (exact)
    s0 = (f32(cx), f32(cy))
    s1 = (f32(cx + 0.0), f32(cy + v))
    d0 = (f32(out_w * 0.5), f32(out_h * 0.5))
    d1 = (d0[0], f32(d0[1] + f32(out_w * -0.5)))

    def third(a, b):                                         # get_3rd_point, in float32
        return (f32(b[0] + f32(-f32(a[1] - b[1]))), f32(b[1] + f32(a[0] - b[0])))
    src = np.array([s0, s1, third(s0, s1)], np.float32)
    dst = np.array([d0, d1, third(d0, d1)], np.float32)
    return src, dst


def get_affine(src, dst):
    """cv2.getAffineTransform(src, dst): the 6x6 system solved by OpenCV's partial-pivot LU (eliminate with
    d = -1/pivot, back-substitute by division); all zeros when a pivot is below LU_EPS, as cv::solve returns."""
    a = np.zeros((6, 6))
    b = np.zeros(6)
    for i in range(3):
        a[2 * i, 0:3] = [float(src[i, 0]), float(src[i, 1]), 1.0]
        a[2 * i + 1, 3:6] = [float(src[i, 0]), float(src[i, 1]), 1.0]
        b[2 * i], b[2 * i + 1] = float(dst[i, 0]), float(dst[i, 1])
    A = a.tolist()
    b = b.tolist()
    for i in range(6):
        k = i
        for j in range(i + 1, 6):
            if abs(A[j][i]) > abs(A[k][i]):
                k = j
        if abs(A[k][i]) < LU_EPS:
            return np.zeros((2, 3))
        if k != i:
            A[i], A[k] = A[k], A[i]
            b[i], b[k] = b[k], b[i]
        d = -1.0 / A[i][i]
        for j in range(i + 1, 6):
            alpha = A[j][i] * d
            for kk in range(i + 1, 6):
                A[j][kk] = A[j][kk] + alpha * A[i][kk]
            b[j] = b[j] + alpha * b[i]
    for i in range(5, -1, -1):
        s = b[i]
        for kk in range(i + 1, 6):
            s = s - A[i][kk] * b[kk]
        b[i] = s / A[i][i]
    return np.array(b).reshape(2, 3)


def crop_matrices(center, scale, out_w, out_h):
    """(forward, inverse) crop matrices: get_affine_transform(..., inv=0) and (..., inv=1)."""
    src, dst = crop_points(center, scale, out_w, out_h)
    return get_affine(src, dst), get_affine(dst, src)


def invert_for_warp(M):
    """warpAffine's own inversion of the forward matrix (D = 0 when singular)."""
    m = [float(x) for x in np.asarray(M, np.float64).ravel()]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    a11, a22 = m[4] * D, m[0] * D
    m[0], m[1], m[3], m[4] = a11, m[1] * -D, m[3] * -D, a22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return m


def _round_int(v):
    """saturate_cast<int>(double): round half to even."""
    return np.rint(v).astype(np.int64)


def warp_linear(img, M, out_w, out_h):
    """cv2.warpAffine(img, M, (out_w, out_h), flags=INTER_LINEAR) with the zero border: 10-bit fixed-point offsets
    rounded half to even, 5-bit sub-pixel positions, 15-bit bilinear weights.  img uint8 [H,W] or [H,W,C]."""
    img = np.asarray(img)
    squeeze = img.ndim == 2
    if squeeze:
        img = img[:, :, None]
    m = invert_for_warp(M)
    H, W, C = img.shape
    xs = np.arange(out_w, dtype=np.float64)
    adelta = _round_int(m[0] * xs * 1024)
    bdelta = _round_int(m[3] * xs * 1024)
    ys = np.arange(out_h, dtype=np.float64)
    X0 = _round_int((m[1] * ys + m[2]) * 1024) + 16
    Y0 = _round_int((m[4] * ys + m[5]) * 1024) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy, fx, fy = X >> 5, Y >> 5, X & 31, Y & 31
    acc = np.zeros((out_h, out_w, C), np.int64)
    for dy, dx, w in ((0, 0, (32 - fy) * (32 - fx)), (0, 1, (32 - fy) * fx), (1, 0, fy * (32 - fx)), (1, 1, fy * fx)):
        yy, xx = sy + dy, sx + dx
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        v = np.zeros((out_h, out_w, C), np.int64)
        v[ok] = img[yy[ok], xx[ok]]
        acc += v * (w * 32)[:, :, None]
    out = np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)
    return out[:, :, 0] if squeeze else out


def dot_affine(pts, M):
    """data_utils.affine_transform(pts, M) = np.dot(pts, M[:, :2].T) + M[:, 2] in float64, with np.dot's x * m0 rounded
    and y * m1 fused into it."""
    pts = np.asarray(pts, np.float64).reshape(-1, 2)
    out = np.empty_like(pts)
    for i, (x, y) in enumerate(pts):
        for j in range(2):
            out[i, j] = _fma(y, M[j, 1], x * M[j, 0]) + M[j, 2]
    return out


def magnify(box, M, ratio, out_w, out_h):
    """magnify_box(affine_transform(box corners, M), ratio, out_h, out_w) -> (x0, y0, x1, y1) inclusive."""
    p = dot_affine(np.asarray(box, np.float64).reshape(2, 2), M)
    mean = (p[0] + p[1]) / 2.0
    r = np.rint((p - mean) * ratio + mean)
    r = np.where(np.abs(r) < 2.0 ** 31, r, -2.0 ** 31).astype(np.int64)        # astype(int32) of an overflow
    r[:, 0] = np.clip(r[:, 0], 0, out_w - 1)
    r[:, 1] = np.clip(r[:, 1], 0, out_h - 1)
    return int(r[0, 0]), int(r[0, 1]), int(r[1, 0]), int(r[1, 1])


def normalise(u8, mean=MEAN, std=STD):
    """(u8 / 255 - mean) / std in float32, HWC -> CHW."""
    x = u8.astype(np.float32) / f32(255.0)
    return ((x - mean.reshape(1, 1, 3)) / std.reshape(1, 1, 3)).transpose(2, 0, 1)


def center_scale(box, scale_ratio, center_f32=True):
    """pvnet_transform's centre (rounded to float32) and scale; the cascade's _crop keeps the centre in float64."""
    b = [float(x) for x in box]
    c = np.array([(b[0] + b[2]) / 2.0, (b[1] + b[3]) / 2.0])
    if center_f32:
        c = c.astype(np.float32).astype(np.float64)
    w, h = b[2] - b[0], b[3] - b[1]
    return c, (h if h > w else w) * scale_ratio


def crop_restated(img, box, input_size=(256, 256), scale_ratio=2.4, box_ratio=1.2, mask_to_box=True, center_f32=True):
    """pvnet_transform(img, box) (mask_to_box=True) or the cascade's _crop (mask_to_box=False, center_f32=False):
    (inp float32 [3,h,w], crop uint8 [h,w,3], center float64 [2], scale float64, forward M, inverse M)."""
    w, h = input_size
    c, s = center_scale(box, scale_ratio, center_f32)
    M, Minv = crop_matrices(c, s, w, h)
    u8 = warp_linear(img, M, w, h)
    if mask_to_box:
        x0, y0, x1, y1 = magnify(box, M, box_ratio, w, h)
        keep = np.zeros_like(u8)
        keep[y0:y1 + 1, x0:x1 + 1] = u8[y0:y1 + 1, x0:x1 + 1]
        u8 = keep
    return normalise(u8), u8, c, s, M, Minv


def uncrop_restated(kpt, center, scale, input_size):
    """affine_transform(kpt [K,2], get_affine_transform(center, scale, 0, input_size, inv=1)) in float64."""
    _, Minv = crop_matrices(center, scale, *input_size)
    return dot_affine(np.asarray(kpt, np.float32), Minv)


# ---- seeded cases --------------------------------------------------------------------------------------------------

def random_boxes(rng, n, W=720, H=540):
    """xyxy float64 boxes of every kind the crop meets: inside, touching and beyond each edge, entirely outside, 2-pixel
    and near-full-image, with integer, half-integer and random-float coordinates."""
    out = []
    for i in range(n):
        kind = i % 8
        if kind == 0:                                   # inside, random float
            w, h = rng.uniform(20, 300, 2)
            x0, y0 = rng.uniform(0, W - w), rng.uniform(0, H - h)
        elif kind == 1:                                 # integer coordinates, touching an edge
            w, h = rng.integers(10, 200, 2).astype(float)
            x0, y0 = [(0.0, rng.integers(0, H - h)), (W - w, rng.integers(0, H - h)),
                      (rng.integers(0, W - w), 0.0), (rng.integers(0, W - w), H - h)][rng.integers(0, 4)]
        elif kind == 2:                                 # half-integer, partly beyond an edge
            w, h = rng.integers(20, 300, 2) + 0.5
            x0, y0 = rng.integers(-150, W - 50) + 0.5, rng.integers(-150, H - 50) + 0.5
        elif kind == 3:                                 # entirely outside
            w, h = rng.uniform(10, 100, 2)
            x0 = rng.choice([rng.uniform(-400, -w - 1), rng.uniform(W + 1, W + 300)])
            y0 = rng.uniform(-200, H + 200)
        elif kind == 4:                                 # 2-pixel box: strong up-sampling
            w, h = 2.0, 2.0
            x0, y0 = float(rng.integers(0, W - 2)), float(rng.integers(0, H - 2))
        elif kind == 5:                                 # near-full image: down-sampling
            w, h = rng.uniform(W - 40, W), rng.uniform(H - 40, H)
            x0, y0 = rng.uniform(0, W - w), rng.uniform(0, H - h)
        elif kind == 6:                                 # tall and thin / wide and flat
            w, h = (rng.uniform(5, 30), rng.uniform(150, 400)) if rng.random() < 0.5 else \
                (rng.uniform(150, 500), rng.uniform(5, 30))
            x0, y0 = rng.uniform(-20, W - w + 20), rng.uniform(-20, H - h + 20)
        else:                                           # random float anywhere, around the image
            w, h = rng.uniform(1, 400, 2)
            x0, y0 = rng.uniform(-100, W), rng.uniform(-100, H)
        out.append([x0, y0, x0 + w, y0 + h])
    return np.array(out, np.float64)


DEGENERATE = np.array([[100.0, 100.0, 100.0, 100.0],     # a point: singular system, all-zero forward matrix
                       [0.0, 0.0, 0.0, 0.0],
                       [300.5, 200.25, 300.5, 200.25]])


def pattern_images(params, W=720, H=540):
    """uint8 [B,H,W,3] from integer parameters [B,3,4]: ramps, a quadratic term and a hashed texture, all in integer
    arithmetic, so the same parameters give the same bytes everywhere and every byte value occurs."""
    yy, xx = np.mgrid[0:H, 0:W].astype(np.int64)
    out = np.empty((len(params), H, W, 3), np.uint8)
    for b, pb in enumerate(np.asarray(params, np.int64)):
        for c, (p0, p1, p2, p3) in enumerate(pb):
            v = (xx * (p0 % 7) + yy * (p1 % 5) + (xx * xx + 3 * yy * yy) // (64 + p2 % 512)
                 + ((xx * 7919 + yy * 104729 + p3) * 2654435761 >> 13) % (1 + p3 % 48))
            out[b, :, :, c] = v & 255
    return out


def random_images(rng, B, W=720, H=540):
    return pattern_images(rng.integers(1, 1 << 16, (B, 3, 4)), W, H)


def sha256(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
