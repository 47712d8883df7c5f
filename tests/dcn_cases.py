"""Shared DCNv2 cases for tests/test_dcn_host.py and tests/test_gpu_dcn.py.

DETECTOR: (C, H, W, C_out) of the 16 DCN calls of DLASeg('dla34', ...) (lib/networks/ct/dla_dcn.py), in call order, at
the T-LESS test input 736x544 (720x540 padded, tless_test_utils.augment), LINEMOD's 640x480 and 512x512; every one is
3x3, stride 1, pad 1, dilation 1, one deformable group.  test_dcn_host.py records them from the unmodified network.
SWEEP: kernel 1x1 / 3x3 / 5x3, stride 1 / 2, pad 0-2, dilation 1 / 2, dg 1 / 2 / 4, C not a multiple of any tile,
H or W = 1.  make_inputs(case, offsets=...) builds seeded inputs; offsets="edges" puts sample points exactly at -1,
in (-1, 0), at 0, at integers, at H-1, at H, far outside and (nonfinite=True) at NaN / +-inf; masks are 0, 1 and
fractions.
"""
from collections import namedtuple

import numpy as np

Case = namedtuple("Case", "B C H W Co kh kw stride pad dil dg")

_DLA = [(512, 1 / 32, 256), (256, 1 / 16, 256), (256, 1 / 16, 128), (128, 1 / 8, 128), (256, 1 / 16, 128),
        (128, 1 / 8, 128), (128, 1 / 8, 64), (64, 1 / 4, 64), (128, 1 / 8, 64), (64, 1 / 4, 64), (128, 1 / 8, 64),
        (64, 1 / 4, 64), (128, 1 / 8, 64), (64, 1 / 4, 64), (256, 1 / 16, 64), (64, 1 / 4, 64)]
INPUTS = {"544x736": (544, 736), "480x640": (480, 640), "512x512": (512, 512)}


def detector_shapes(key):
    h, w = INPUTS[key]
    return [(c, int(h * f), int(w * f), co) for c, f, co in _DLA]


DETECTOR = {key: [Case(1, c, h, w, co, 3, 3, (1, 1), (1, 1), (1, 1), 1) for c, h, w, co in detector_shapes(key)]
            for key in INPUTS}

SWEEP = [
    Case(2, 5, 7, 9, 3, 3, 3, (1, 1), (1, 1), (1, 1), 1),
    Case(2, 8, 9, 6, 5, 3, 3, (2, 2), (1, 1), (1, 1), 2),
    Case(1, 12, 8, 8, 7, 5, 3, (1, 2), (2, 1), (1, 1), 4),
    Case(2, 4, 10, 11, 6, 3, 3, (1, 1), (2, 2), (2, 2), 1),
    Case(1, 6, 6, 5, 4, 1, 1, (1, 1), (0, 0), (1, 1), 2),
    Case(2, 3, 1, 9, 4, 1, 3, (1, 1), (0, 1), (1, 1), 1),
    Case(1, 4, 9, 1, 3, 3, 1, (2, 1), (1, 0), (1, 1), 4),
    Case(1, 20, 5, 7, 9, 3, 3, (1, 1), (0, 0), (1, 2), 4),
    Case(3, 17, 13, 12, 70, 3, 3, (1, 1), (1, 1), (1, 1), 1),
    Case(1, 130, 6, 9, 33, 3, 3, (2, 1), (1, 2), (1, 1), 2),
]


def case_id(c):
    return (f"B{c.B}C{c.C}H{c.H}W{c.W}o{c.Co}k{c.kh}x{c.kw}s{c.stride[0]}{c.stride[1]}p{c.pad[0]}{c.pad[1]}"
            f"d{c.dil[0]}{c.dil[1]}g{c.dg}")


def out_hw(c):
    return ((c.H + 2 * c.pad[0] - (c.dil[0] * (c.kh - 1) + 1)) // c.stride[0] + 1,
            (c.W + 2 * c.pad[1] - (c.dil[1] * (c.kw - 1) + 1)) // c.stride[1] + 1)


def _edge_offsets(c, rng, nonfinite):
    """Offsets that put the sample point of every tap at one of the edge positions of its axis."""
    Ho, Wo = out_hw(c)
    T = c.kh * c.kw
    ii, jj = np.divmod(np.arange(T), c.kw)
    base_h = (np.arange(Ho)[None, :, None] * c.stride[0] - c.pad[0] + ii[:, None, None] * c.dil[0]).astype(np.float32)
    base_w = (np.arange(Wo)[None, None, :] * c.stride[1] - c.pad[1] + jj[:, None, None] * c.dil[1]).astype(np.float32)

    def targets(n):
        t = [-1.0, -0.5, -1e-3, 0.0, 1.0, n - 1.0, n - 1.0 + 0.25, float(n), n + 0.5, -40.0, 1e6, 0.5, 2.75]
        if nonfinite:
            t += [np.nan, np.inf, -np.inf]
        return np.array(t, np.float32)

    th, tw = targets(c.H), targets(c.W)
    shp = (c.B, c.dg, T, Ho, Wo)
    want_h = th[rng.integers(0, len(th), shp)]
    want_w = tw[rng.integers(0, len(tw), shp)]
    with np.errstate(invalid="ignore", over="ignore"):
        dy = (want_h - base_h[None, None]).astype(np.float32)
        dx = (want_w - base_w[None, None]).astype(np.float32)
    off = np.stack([dy, dx], axis=3)                  # [B, dg, T, 2, Ho, Wo]
    return off.reshape(c.B, c.dg * 2 * T, Ho, Wo)


def make_inputs(c, seed=0, offsets="random", nonfinite=False):
    """(input, offset, mask, weight, bias) as float32 numpy arrays.  offsets: "random" (|offset| < 2.5, non-integer
    sample points), "edges" (see the module docstring) or "zero"."""
    rng = np.random.default_rng(seed)
    Ho, Wo = out_hw(c)
    T = c.kh * c.kw
    x = rng.standard_normal((c.B, c.C, c.H, c.W)).astype(np.float32)
    if offsets == "edges":
        off = _edge_offsets(c, rng, nonfinite)
    elif offsets == "zero":
        off = np.zeros((c.B, c.dg * 2 * T, Ho, Wo), np.float32)
    else:
        off = rng.uniform(-2.5, 2.5, (c.B, c.dg * 2 * T, Ho, Wo)).astype(np.float32)
        frac = off - np.floor(off)
        off = np.where(np.abs(frac - 0.5) > 0.49, off + 0.02, off)                        # keep off integer points
        off = (np.round(off * 1024) / 1024).astype(np.float32)     # so float(base) + offset is exact in fp32
    mask = rng.uniform(0, 1, (c.B, c.dg * T, Ho, Wo)).astype(np.float32)
    sel = rng.integers(0, 4, mask.shape)
    mask = np.where(sel == 0, 0.0, np.where(sel == 1, 1.0, mask)).astype(np.float32)
    w = (rng.standard_normal((c.Co, c.C, c.kh, c.kw)) / np.sqrt(c.C * T)).astype(np.float32)
    b = rng.standard_normal(c.Co).astype(np.float32)
    return x, off, mask, w, b


def identity_weight(c):
    """W[o, c, i, j] = [o == c*kh*kw + i*kw + j], C_out = C*kh*kw: the forward then returns the columns exactly."""
    K = c.C * c.kh * c.kw
    return np.eye(K, dtype=np.float32).reshape(K, c.C, c.kh, c.kw), np.zeros(K, np.float32)
