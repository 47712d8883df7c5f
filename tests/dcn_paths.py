"""DCNv2 cases that reach every load path and tile tail of csrc/dcn.cu's half-precision forward, and a twin of the launch
decisions that select them, for tests/test_dcn_paths_host.py and tests/test_gpu_dcn_paths.py.

forward_half_body<T, NHWC> picks its path from the shape: the weight tile arrives by 16-byte cp.async when every group
is a multiple of 8 channels wide (`vec`), the NHWC sampler reads 8 channels of a corner in one 16-byte load when the
input is also 16-byte aligned (`vin`), the last K chunk of a group is partial when the group is not a multiple of 32
channels wide (`tail`), warps whose 32 rows lie past C_out skip the MMAs (`live`), and dcn_half_splits spreads the K
chunks over a cluster of S CTAs.  The detector's layers all take the same side of each of these, so PATHS picks small
shapes (H, W <= 16, B <= 5: the fp64 restatement takes milliseconds) that between them take every side: cells()
names the sides one forward run takes, and REQUIRED lists them all.  BACKWARD adds the fp32 backward's grad_weight
channel tiles (BN = 128 channels of a group per tile).

The GPU tests run each PATHS case in both layouts (LAYOUTS), and each once more on a channels_last input whose data
pointer is 2 bytes past a 16-byte boundary, which turns `vin` off and leaves `vec` on.
"""
import dcn_cases as dc
from dcn_cases import Case

# dcn.cu's tile and split constants, restated; test_dcn_paths_host.py checks them against the source
H_TARGET_CTAS, H_MAX_SPLIT, H_MIN_CHUNKS = 264, 8, 4
HBM, HBN, HBK = 128, 64, 32
BN = 128                     # the fp32 grad_weight kernel's channel tile

LAYOUTS = ("nchw", "channels_last")


def _cg(c):
    return c.C // c.dg


def _nct(c):
    return (_cg(c) + HBK - 1) // HBK


def nchunk(c):
    """K chunks of one image: (group, tap, 32-channel chunk of the group)."""
    return c.dg * c.kh * c.kw * _nct(c)


def half_splits(c):
    """dcn_half_splits, line for line: the split-K factor S of the half-precision forward."""
    T = c.kh * c.kw
    Cg = c.C // c.dg
    n = c.dg * T * ((Cg + HBK - 1) // HBK)
    Ho, Wo = dc.out_hw(c)
    tiles = (Ho * Wo + HBN - 1) // HBN * ((c.Co + HBM - 1) // HBM)
    S = (H_TARGET_CTAS + tiles - 1) // tiles
    if S > H_MAX_SPLIT:
        S = H_MAX_SPLIT
    if S > n // H_MIN_CHUNKS:
        S = n // H_MIN_CHUNKS
    return 1 if S < 1 else S


def grid(c):
    """The half-precision forward's launch grid: (ceil(P / HBN) * S, ceil(C_out / HBM), B)."""
    Ho, Wo = dc.out_hw(c)
    return ((Ho * Wo + HBN - 1) // HBN * half_splits(c), otiles(c), c.B)


def vec(c):
    """The weight tile arrives by 16-byte cp.async: (C | C/dg) % 8 == 0 (the tap-major weight the Python layer passes
    is always 16-byte aligned)."""
    return ((c.C | _cg(c)) & 7) == 0


def tail(c):
    """Channels in the last, partial K chunk of a group (0: every chunk is full)."""
    return _cg(c) % HBK


def otiles(c):
    return (c.Co + HBM - 1) // HBM


def live_warps_in_last_tile(c):
    """Warp rows (of 4, 32 output channels each) of the last output tile that hold a channel: the others are not
    `live` and skip the MMAs."""
    return (c.Co - (otiles(c) - 1) * HBM + 31) // 32


def split_starts(c):
    """(group, tap, first channel) of each cluster rank's first K chunk kb = r * nchunk / S."""
    T, nct, n, S = c.kh * c.kw, _nct(c), nchunk(c), half_splits(c)
    out = []
    for r in range(S):
        kb = r * n // S
        out.append((kb // (T * nct), (kb // nct) % T, (kb % nct) * HBK))
    return out


def cells(c, layout, aligned=True):
    """The sides of forward_half_body's branches one forward run of case c takes."""
    s = set()
    if not vec(c):
        if c.C % 8 == 0:
            s.add("scalar weight tile with C % 8 == 0")
        return s
    s.add(f"vec dg={c.dg}")
    s.add(f"vec tail={tail(c)}")
    s.add(f"vec S={half_splits(c)}")
    if c.Co % HBM and otiles(c) > 1:
        s.add(f"vec {otiles(c)} output tiles, {live_warps_in_last_tile(c)} live warps in the last")
    for r, (g, tap, c0) in enumerate(split_starts(c)):
        if r and g > 0 and (tap, c0) != (0, 0):
            s.add("vec split starts mid-group, g > 0")
        if r and g > 0 and c0 > 0:
            s.add("vec split starts mid-tap, g > 0")
    if max(c.stride) > 1:
        s.add("vec stride > 1")
    if c.pad != (1, 1):
        s.add("vec pad != 1")
    if max(c.dil) > 1:
        s.add("vec dilation > 1")
    if layout == "channels_last":
        s.add("vin: 16-byte NHWC corner loads" if aligned else "scalar NHWC sampler with C % 8 == 0")
    return s


_BOTH = ([f"vec dg={g}" for g in (1, 2, 4)] + [f"vec tail={t}" for t in (0, 8, 16, 24)] +
         ["scalar weight tile with C % 8 == 0"] +
         [f"vec {ot} output tiles, {lw} live warps in the last" for ot, lw in ((2, 1), (2, 3), (3, 1))] +
         [f"vec S={s}" for s in range(1, 9)] +
         ["vec split starts mid-group, g > 0", "vec split starts mid-tap, g > 0",
          "vec stride > 1", "vec pad != 1", "vec dilation > 1"])
REQUIRED = ({(name, lay) for name in _BOTH for lay in LAYOUTS} |
            {("vin: 16-byte NHWC corner loads", "channels_last"),
             ("scalar NHWC sampler with C % 8 == 0", "channels_last")})


def reached(cases):
    """(cell, layout) of every run the GPU tests make of cases: each in both layouts, and channels_last misaligned."""
    out = set()
    for c in cases:
        for lay in LAYOUTS:
            out |= {(name, lay) for name in cells(c, lay)}
        out |= {(name, "channels_last") for name in cells(c, "channels_last", aligned=False)}
    return out


# Each comment: C / dg = group width -> tail, nchunk -> S (one or a few pixel tiles, so S = min(8, nchunk // 4)).
PATHS = [
    Case(2, 48, 9, 7, 129, 1, 1, (1, 1), (0, 0), (1, 1), 2),     # 24 -> 24; 2 -> S=1; C_out 129
    Case(3, 32, 10, 12, 64, 3, 3, (1, 1), (1, 1), (1, 1), 1),    # 32 -> 0; 9 -> S=2; two pixel tiles
    Case(1, 24, 11, 9, 40, 5, 3, (2, 1), (2, 1), (1, 1), 1),     # 24 -> 24; 15 -> S=3; stride 2
    Case(2, 16, 7, 9, 200, 3, 3, (1, 1), (1, 1), (1, 1), 2),     # 8 -> 8; 18 -> S=4, rank 3 starts mid-group 1
    Case(2, 64, 8, 8, 257, 1, 5, (1, 1), (0, 2), (1, 1), 4),     # 16 -> 16; 20 -> S=5; C_out 257
    Case(1, 64, 9, 10, 48, 2, 3, (1, 1), (1, 1), (2, 1), 4),     # 16 -> 16; 24 -> S=6; dilation 2
    Case(2, 56, 12, 12, 33, 5, 3, (1, 1), (2, 1), (1, 1), 1),    # 56 -> 24; 30 -> S=7, a rank starts mid-tap
    Case(2, 80, 8, 9, 72, 3, 3, (1, 1), (1, 1), (1, 1), 2),      # 40 -> 8; 36 -> S=8, rank 6 starts mid-tap of group 1
    Case(2, 24, 7, 8, 20, 3, 3, (1, 1), (1, 1), (1, 1), 2),      # 12: C % 8 == 0 but not the group, no vec
]

# the fp32 backward's grad_weight tiles a group's channels by BN = 128: two tiles, the second holding 8 channels, and
# three, the third holding 1
GW_TILES = [
    Case(3, 272, 5, 6, 70, 3, 3, (1, 1), (1, 1), (1, 1), 2),
    Case(3, 257, 5, 4, 12, 3, 3, (1, 1), (1, 1), (1, 1), 1),
]
BACKWARD = PATHS + GW_TILES
BACKWARD_BATCHES = (3, 5)     # run once in one grad_cols chunk and once in chunks of 2 images: a partial last chunk


def grad_weight_tiles(c):
    """(channel tiles of a group, channels in the last) of dcn_grad_weight_kernel."""
    Cg = _cg(c)
    n = (Cg + BN - 1) // BN
    return n, Cg - (n - 1) * BN


def column_entries(c):
    """Entries of the column matrix [B, C*kh*kw, Ho*Wo]: the fp64 restatement's working size."""
    Ho, Wo = dc.out_hw(c)
    return c.B * c.C * c.kh * c.kw * Ho * Wo
