"""Shared by tests/test_render_host.py and tests/test_gpu_render.py: a numpy restatement of T-LESS's VSD (as
Evaluator.vsd_metric computes it, lib/evaluators/tless_test/pvnet.py:66-105 over lib/utils/vsd) and the synthetic meshes
and poses the renderer is checked on.  Meshes are in millimetres, like the evaluator's model."""
import numpy as np

DELTA, TAU, THRESHOLD = 15, 20, 0.3
# T-LESS's Primesense intrinsics (720 x 540) and a 128 x 128 camera
K_TLESS = np.array([[1075.65091572, 0.0, 367.06888344], [0.0, 1073.90347929, 247.72159802], [0.0, 0.0, 1.0]])
K_SMALL = np.array([[190.0, 0.0, 63.3], [0.0, 187.5, 64.1], [0.0, 0.0, 1.0]])


def dist_im(depth, K):
    """misc.depth_im_to_dist_im: ((c - cx) * Z) * (1 / fx), likewise for rows, then sqrt((X*X + Y*Y) + Z*Z) in fp64."""
    H, W = depth.shape
    z = depth.astype(np.float64)
    X = ((np.arange(W, dtype=np.float64)[None, :] - K[0, 2]) * z) * (1.0 / K[0, 0])
    Y = ((np.arange(H, dtype=np.float64)[:, None] - K[1, 2]) * z) * (1.0 / K[1, 1])
    return np.sqrt((X * X + Y * Y) + z * z)


def vsd_restated(depth_est, depth_gt, depth_test, K, delta=DELTA, tau=TAU):
    """vsd_utils.vsd with the 'step' cost on the distance images and visibility masks vsd_metric builds."""
    dt, dg, de = (dist_im(d, K) for d in (depth_test, depth_gt, depth_est))
    f32, fd = np.float32, np.float32(delta)
    vg = (dt > 0) & (dg > 0) & (dg.astype(f32) - dt.astype(f32) <= fd)
    ve = ((dt > 0) & (de > 0) & (de.astype(f32) - dt.astype(f32) <= fd)) | (vg & (de > 0))
    inter, union = vg & ve, vg | ve
    nu, ni = int(union.sum()), int(inter.sum())
    nc = int((inter & (np.abs(dg - de) >= tau)).sum())
    return (nc + nu - ni) / float(nu) if nu else 1.0


def vsd_metric_restated(depth_of, poses_est, poses_gt, K, depth_test):
    """Evaluator.vsd_metric's flag: 1 when any (estimate, ground truth) pair has e < 0.3.  depth_of(pose) renders."""
    for pe in poses_est:
        de = depth_of(pe)
        for pg in poses_gt:
            if vsd_restated(de, depth_of(pg), depth_test, K) < THRESHOLD:
                return 1
    return 0


# ---- meshes ---------------------------------------------------------------------------------------------------------

def box(sx=60.0, sy=40.0, sz=50.0):
    v = np.array([[x, y, z] for x in (-sx, sx) for y in (-sy, sy) for z in (-sz, sz)], np.float64)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
                  [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    return v.astype(np.float32), f


def icosphere(subdiv=5, r=55.0):
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    for _ in range(subdiv):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return (np.array(v) * r).astype(np.float32), np.array(f, np.int32)


def torus(R=50.0, r=18.0, nu=96, nv=48):
    u, v = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    pts = np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    c, d = ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
    f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return pts.astype(np.float32), f.astype(np.int32)


def soup(nf, seed=0, extent=80.0, size=4.0):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-extent, extent, (nf, 1, 3))
    pts = (c + rng.normal(0, size, (nf, 3, 3))).reshape(-1, 3)
    return pts.astype(np.float32), np.arange(3 * nf, dtype=np.int32).reshape(nf, 3)


MESHES = {"box": box, "icosphere": icosphere, "torus": torus, "soup100k": lambda: soup(100_000)}
CLOSED = ("box", "icosphere", "torus")


def rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def poses(n, seed, z=(550.0, 900.0), xy=60.0):
    """n random [R|t] in millimetres in front of the camera."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 3, 4))
    for i in range(n):
        out[i, :, :3] = rotation(rng)
        out[i, :, 3] = (rng.uniform(-xy, xy), rng.uniform(-xy, xy), rng.uniform(*z))
    return out
