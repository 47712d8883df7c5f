"""Seeded clouds for the farthest-point-sampling tests, a numpy restatement of the reference loop
(lib/csrc/fps/src/farthest_point_sampling.cpp) and a ctypes loader for the reference build oracle/_ref/libfps_ref.so.

The fixture tests/golden/fps.npz stores each case's (kind, pn, sn, seed, init_center, start) and the reference's indices;
`cloud(kind, pn, seed)` rebuilds the points."""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libfps_ref.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "fps.npz")
FLT_MAX = np.float32(np.finfo(np.float32).max)

# normal: Gaussian; lattice: integer coordinates in [-4, 4], so many distances tie exactly across CTAs and cluster ranks;
# dup: a quarter as many distinct points, each repeated; same: one point pn times; nanf: Gaussian with NaN and +-inf
KINDS = ("normal", "lattice", "dup", "same", "nanf")

# the kernel's boundaries: a warp (32), a CTA's threads (512), a CTA's on-chip slice (8192 points), clusters of 2, 4, 8
# CTAs (16384, 32768, 65536 points on chip) and the streamed remainder beyond them
BOUNDARY_PN = (511, 512, 513, 8191, 8192, 8193, 16384, 16385, 32768, 32769, 65536, 65537)


def cases():
    """(kind, pn, sn, seed) of the fixture; each runs in both modes."""
    out = []
    seed = 1000
    for pn in (1, 2, 31, 32, 33, 1000):
        for sn in sorted({0, 1, 8, 64, pn, pn + 3}):
            out.append(("normal", pn, sn, seed)); seed += 1
    for pn in BOUNDARY_PN:
        out.append(("normal", pn, 64, seed)); seed += 1
        out.append(("lattice", pn, 64, seed)); seed += 1
    for pn, sn in ((100000, 8), (100000, 64), (1000000, 8)):
        out.append(("normal", pn, sn, seed)); seed += 1
    for pn, sn in ((1000, 300), (8193, 200), (40000, 300), (70000, 100)):
        out.append(("lattice", pn, sn, seed)); seed += 1
    for kind in ("dup", "same", "nanf"):
        for pn in (33, 1000, 20000):
            for sn in ((8, 64, pn + 3) if pn < 20000 else (8, 64)):
                out.append((kind, pn, sn, seed)); seed += 1
    return out


def cloud(kind, pn, seed):
    rng = np.random.default_rng(seed)
    if kind == "normal":
        return rng.standard_normal((pn, 3)).astype(np.float32)
    if kind == "lattice":
        return rng.integers(-4, 5, (pn, 3)).astype(np.float32)
    if kind == "dup":
        base = rng.standard_normal((max(1, pn // 4), 3)).astype(np.float32)
        return base[rng.integers(0, len(base), pn)]
    if kind == "same":
        return np.repeat(rng.standard_normal((1, 3)).astype(np.float32), pn, axis=0)
    if kind == "nanf":
        p = rng.standard_normal((pn, 3)).astype(np.float32)
        flat = p.reshape(-1)
        k = max(1, flat.size // 16)
        flat[rng.choice(flat.size, k, replace=False)] = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), k)
        return p
    raise ValueError(kind)


def fps_restated(pts, sn, start=None):
    """The reference loop in numpy float32 (each product and sum rounded on its own, as gcc -O2 without -march computes
    it).  start=None is farthest_point_sampling_init_center; otherwise the random variant from `start`."""
    p = np.ascontiguousarray(pts, np.float32)
    pn = len(p)

    def sq(q):
        d = p - q
        return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]

    mask = np.zeros(pn, bool)

    def argmax(md):
        v = np.where(mask | ~(md > 0), np.float32(-1), md)
        i = int(np.argmax(v))
        return i if v[i] > 0 else 0

    if start is None:
        with np.errstate(invalid="ignore"):
            mx = np.array([max(-FLT_MAX, np.nanmax(c)) if not np.isnan(c).all() else -FLT_MAX for c in p.T], np.float32)
            mn = np.array([min(FLT_MAX, np.nanmin(c)) if not np.isnan(c).all() else FLT_MAX for c in p.T], np.float32)
            centre = (mx + mn) * np.float32(0.5)
            d = sq(centre)
            md = np.where(FLT_MAX < d, FLT_MAX, d).astype(np.float32)
        cur = argmax(md)
    else:
        md = np.full(pn, FLT_MAX, np.float32)
        cur = int(start)
    out = np.zeros(sn, np.int32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(sn):
            mask[cur] = True
            out[i] = cur
            if i < sn - 1:
                d = sq(p[cur])
                md = np.where(~mask & (d < md), d, md)
                cur = argmax(md)
    return out


def ref_lib():
    """The reference build (oracle/_ref/libfps_ref.so) or None when it was not built."""
    if not os.path.exists(REF_LIB):
        return None
    lib = ctypes.CDLL(REF_LIB)
    for name in ("farthest_point_sampling", "farthest_point_sampling_init_center"):
        fn = getattr(lib, name)
        fn.restype = None
        fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    return lib


def ref_fps(lib, pts, sn, init_center):
    """The reference's indices; the random variant draws its own start (its idxs[0] when sn > 0)."""
    p = np.ascontiguousarray(pts, np.float32)
    idxs = np.zeros(sn, np.int32)
    fn = lib.farthest_point_sampling_init_center if init_center else lib.farthest_point_sampling
    fn(p.ctypes.data, idxs.ctypes.data, len(p), sn)
    return idxs


def load_golden():
    """[(kind, pn, sn, seed, init_center, start, idxs)] from tests/golden/fps.npz."""
    z = np.load(GOLDEN)
    out = []
    for k in range(len(z["pn"])):
        lo, hi = int(z["offset"][k]), int(z["offset"][k + 1])
        out.append((KINDS[int(z["kind"][k])], int(z["pn"][k]), int(z["sn"][k]), int(z["seed"][k]),
                    bool(z["init_center"][k]), int(z["start"][k]), z["idxs"][lo:hi]))
    return out
