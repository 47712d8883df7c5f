"""Shared by tests/test_tless_masks_host.py, tests/test_gpu_tless_masks.py and tests/golden/make_golden_tless_masks.py: the
seeded depth stacks T-LESS's instance masks are checked on, and a numpy restatement of what
lib/datasets/tless/handle_test_data.py builds from them (get_mask's update_mask loop over opengl_renderer.render's
depth / 1000, the pixel_num.pkl count, and the visible-mask count and cv2.boundingRect test_to_coco takes)."""
import numpy as np

LABEL_BG = 0


def compose_restated(depth_mm, obj_ids):
    """One image: depth_mm [m,H,W] fp32 in mm (the renderer's depth), obj_ids [m].  Returns (label int16 [H,W],
    a_pixel_num [m], pixel_num [m], bbox [m,4] (x, y, w, h)) as int64 arrays."""
    depth_mm = np.asarray(depth_mm, np.float32)
    m, H, W = depth_mm.shape
    label = np.zeros((H, W), np.int16)
    depth_map = np.full((H, W), 10.0, np.float32)
    a = np.zeros(m, np.int64)
    win = np.full((H, W), -1, np.int64)
    for j in range(m):
        key = depth_mm[j] / np.float32(1000.0)          # opengl_renderer.render: fp32 depth / 1000. stays fp32
        rendered = key != 0
        a[j] = int(rendered.sum())
        take = rendered & (key < depth_map)
        label[take] = int(obj_ids[j]) * 1000 + j
        depth_map[take] = key[take]
        win[take] = j
    p = np.zeros(m, np.int64)
    box = np.zeros((m, 4), np.int64)
    for j in range(m):
        ys, xs = np.nonzero(win == j)
        p[j] = len(xs)
        if len(xs):
            box[j] = (xs.min(), ys.min(), xs.max() - xs.min() + 1, ys.max() - ys.min() + 1)
    return label, a, p, box


def _same_key_pair(rng):
    """Two different fp32 mm depths whose fp32 metre keys are equal."""
    while True:
        d = np.float32(rng.uniform(400, 2000))
        e = np.nextafter(d, np.float32(np.inf))
        if d / np.float32(1000) == e / np.float32(1000):
            return d, e


def _blob(rng, H, W, cover=0.35):
    """A random ellipse mask covering up to about `cover` of the image."""
    cy, cx = rng.uniform(0, H), rng.uniform(0, W)
    ry, rx = rng.uniform(0.1, cover) * H + 1, rng.uniform(0.1, cover) * W + 1
    y, x = np.mgrid[:H, :W]
    return ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2 <= 1


def _surface(rng, H, W, lo=500.0, hi=1500.0, step=0.5):
    """A tilted plane of mm depths on a `step` grid, so neighbouring instances tie often."""
    y, x = np.mgrid[:H, :W]
    z = rng.uniform(lo, hi) + rng.uniform(-0.4, 0.4) * x + rng.uniform(-0.4, 0.4) * y
    return (np.round(z / step) * step).astype(np.float32)


def cases(seed=20261017):
    """[(name, depth_mm [m,H,W] fp32, obj_ids [m] int)] for one image each."""
    rng = np.random.default_rng(seed)
    out = []

    def random_image(name, H, W, m, step=0.5):
        d = np.zeros((m, H, W), np.float32)
        for j in range(m):
            mask = _blob(rng, H, W)
            d[j][mask] = _surface(rng, H, W, step=step)[mask]
        out.append((name, d, rng.integers(1, 31, m)))
        return d

    H, W = 37, 53                                               # not a multiple of 32 either way
    # equal mm depths across instances: the earlier instance keeps every tied pixel
    d = np.zeros((3, H, W), np.float32)
    d[0, 5:30, 4:40] = 800.0
    d[1, 10:35, 10:50] = 800.0
    d[2, 0:20, 20:53] = 800.0
    out.append(("equal_depths", d, np.array([3, 3, 7])))
    # distinct mm depths with one metre key: still a tie, decided by order
    k0, k1 = _same_key_pair(rng)
    d = np.zeros((2, H, W), np.float32)
    d[0, 3:25, 3:30] = k1                                       # the larger mm depth first
    d[1, 10:33, 15:45] = k0
    out.append(("same_key", d, np.array([12, 12])))
    # exactly 10000 mm: key 10.0, counted as rendered but never labelled; beside it, a near instance
    d = np.zeros((3, H, W), np.float32)
    d[0, :, :] = 10000.0
    d[1, 4:20, 4:20] = np.float32(9999.5)
    d[2, 15:30, 10:50] = 10000.0
    out.append(("far_plane", d, np.array([1, 2, 30])))
    # fully occluded and zero-pixel instances
    d = np.zeros((4, H, W), np.float32)
    d[0, 2:30, 2:45] = 600.0
    d[1, 10:20, 10:20] = 900.0                                  # entirely behind instance 0
    d[3, 12:18, 30:40] = 600.0                                  # a tie behind instance 0: also fully occluded
    out.append(("occluded_and_empty", d, np.array([5, 6, 7, 8])))
    # one instance, the whole range of the renderer's depths
    d = np.zeros((1, H, W), np.float32)
    d[0] = rng.uniform(10, 10000, (H, W)).astype(np.float32)
    d[0][rng.random((H, W)) < 0.3] = 0
    out.append(("single", d, np.array([30])))
    # a single-pixel instance at each corner
    d = np.zeros((4, H, W), np.float32)
    for j, (y, x) in enumerate(((0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1))):
        d[j, y, x] = 700.0 + j
    out.append(("corners", d, np.array([1, 2, 3, 4])))
    random_image("random_8", H, W, 8)
    random_image("random_20", 61, 83, 20, step=2.0)
    random_image("random_20_coarse", 33, 31, 20, step=50.0)
    random_image("tless_size_3", 540, 720, 3, step=1.0)
    random_image("tless_size_1", 540, 720, 1, step=1.0)
    return out
