"""ctypes front-end of the CPU oracle (oracle/pvnet_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of pvnet_oracle.c.  Imported by
tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / reference legs;
never by the product package.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

_f32p = ctypes.POINTER(ctypes.c_float)
_i32p = ctypes.POINTER(ctypes.c_int32)
_i64p = ctypes.POINTER(ctypes.c_int64)
_u8p = ctypes.POINTER(ctypes.c_uint8)
_u32p = ctypes.POINTER(ctypes.c_uint32)


def build(force=False):
    so = os.path.join(_HERE, "libpvnet_oracle.so")
    src = os.path.join(_HERE, "pvnet_oracle.c")
    if force or not os.path.exists(so) or (os.path.exists(src) and os.path.getmtime(src) > os.path.getmtime(so)):
        subprocess.check_call(["make", "-C", _HERE, "-B", "libpvnet_oracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libpvnet_oracle.so")
        if not os.path.exists(so):
            build()
        _LIB = ctypes.CDLL(so)
    return _LIB


def _p(a, ty):
    return None if a is None else a.ctypes.data_as(ty)


def _c(a, dt):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


def philox4x32_10(ctr, key):
    c = np.asarray(ctr, dtype=np.uint32)
    k = np.asarray(key, dtype=np.uint32)
    o = np.zeros(4, dtype=np.uint32)
    lib().orc_philox4x32_10(_p(c, _u32p), _p(k, _u32p), _p(o, _u32p))
    return o


def generate_hypothesis(direct, coords, idxs, vanishing_point=False):
    direct = _c(direct, np.float32); coords = _c(coords, np.float32); idxs = _c(idxs, np.int32)
    tn, vn, _ = direct.shape
    hn = idxs.shape[0]
    hyp = np.zeros((hn, vn, 3 if vanishing_point else 2), dtype=np.float32)
    fn = lib().orc_generate_hypothesis_vp if vanishing_point else lib().orc_generate_hypothesis
    fn(_p(direct, _f32p), _p(coords, _f32p), _p(idxs, _i32p), _p(hyp, _f32p), tn, vn, hn)
    return hyp


def voting_for_hypothesis(direct, coords, hyp, inliers, thresh, vanishing_point=False):
    direct = _c(direct, np.float32); coords = _c(coords, np.float32); hyp = _c(hyp, np.float32)
    assert inliers.dtype == np.uint8 and inliers.flags.c_contiguous
    tn, vn, _ = direct.shape
    hn = hyp.shape[0]
    fn = lib().orc_voting_for_hypothesis_vp if vanishing_point else lib().orc_voting_for_hypothesis
    fn(_p(direct, _f32p), _p(coords, _f32p), _p(hyp, _f32p), _p(inliers, _u8p), tn, vn, hn, ctypes.c_float(thresh))
    return inliers


def vote_count(direct, coords, hyp, thresh):
    direct = _c(direct, np.float32); coords = _c(coords, np.float32); hyp = _c(hyp, np.float32)
    tn, vn, _ = direct.shape
    hn = hyp.shape[0]
    counts = np.zeros((hn, vn), dtype=np.int32)
    lib().orc_vote_count(_p(direct, _f32p), _p(coords, _f32p), _p(hyp, _f32p), _p(counts, _i32p),
                         tn, vn, hn, ctypes.c_float(thresh))
    return counts


def select_pixels(mask, mode=0, min_num=5, max_num=30000, selection=None, seed=0, img_base=0, tag=None):
    """Pixel selection of ransac_voting_gpu.py:125-143 (mode 0: v3, `mask.byte()`, fg = sum of byte values) or
    :207-227 (mode 1: distribution, `mask == 1`).  mask int64 [B,H,W]; selection optional float [B,H,W]; without it
    thinning draws from the philox stream (seed, tag, img_base + b), tag defaulting to 2 (v3) / 4 (distribution).
    Returns dict(fg int64 [B], nz int32 [B] (selected before thinning), tn int32 [B] (-1: skipped),
    pix: list of B int32 arrays of row-major pixel indices)."""
    mask = _c(mask, np.int64); selection = _c(selection, np.float32)
    B, H, W = mask.shape
    if selection is not None:
        assert selection.shape == (B, H, W)
    if tag is None:
        tag = 2 if mode == 0 else 4
    fg = np.zeros(B, dtype=np.int64)
    nz = np.zeros(B, dtype=np.int32)
    tn = np.zeros(B, dtype=np.int32)
    pix = np.zeros((B, H * W), dtype=np.int32)
    lib().orc_select_pixels(_p(mask, _i64p), B, H, W, int(mode), int(min_num), int(max_num), _p(selection, _f32p),
                            ctypes.c_uint64(seed), int(img_base), ctypes.c_uint32(tag),
                            _p(fg, _i64p), _p(nz, _i32p), _p(tn, _i32p), _p(pix, _i32p))
    return dict(fg=fg, nz=nz, tn=tn, pix=[pix[b, :max(int(tn[b]), 0)].copy() for b in range(B)])


def ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                           min_num=5, max_num=30000, idxs=None, selection=None, seed=0, img_base=0,
                           debug=False):
    """Oracle twin of ransac_voting_gpu.py:112 (numpy in, numpy out).  `confidence`/`max_iter` do not
    influence the result (see pvnet_oracle.c)."""
    mask = _c(mask, np.int64); vertex = _c(vertex, np.float32)
    B, H, W, K, _ = vertex.shape
    hn = int(round_hyp_num)
    idxs = _c(idxs, np.int32); selection = _c(selection, np.float32)
    if idxs is not None:
        assert idxs.shape == (B, hn, K, 2)
    out = np.zeros((B, K, 2), dtype=np.float32)
    tn = np.zeros(B, dtype=np.int32)
    hyp = np.zeros((B, K, hn, 2), dtype=np.float32) if debug else None
    cnt = np.zeros((B, K, hn), dtype=np.int32) if debug else None
    win = np.zeros((B, K, 2), dtype=np.float32) if debug else None
    rc = lib().orc_ransac_voting_v3(_p(mask, _i64p), _p(vertex, _f32p), B, H, W, K, hn,
                                    ctypes.c_float(inlier_thresh), int(min_num), int(max_num),
                                    _p(idxs, _i32p), _p(selection, _f32p), ctypes.c_uint64(seed), int(img_base),
                                    _p(out, _f32p), _p(tn, _i32p), _p(hyp, _f32p), _p(cnt, _i32p), _p(win, _f32p))
    assert rc == 0
    if debug:
        return out, dict(tn=tn, hyp=hyp, counts=cnt, win=win)
    return out


def estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=256, min_hyp_num=4096, topk=128,
                                           inlier_thresh=0.99, min_num=5, max_num=30000, output_hyp=False,
                                           idxs=None, selection=None, seed=0, img_base=0, debug=False):
    mask = _c(mask, np.int64); vertex = _c(vertex, np.float32); mean = _c(mean, np.float32)
    B, H, W, K, _ = vertex.shape
    hn_total = int(round_hyp_num) * int(np.ceil(min_hyp_num / round_hyp_num))
    idxs = _c(idxs, np.int32); selection = _c(selection, np.float32)
    if idxs is not None:
        assert idxs.shape == (B, hn_total, K, 2)
    cov = np.zeros((B, K, 2, 2), dtype=np.float32)
    hyp = np.zeros((B, K, hn_total, 2), dtype=np.float32) if debug else None
    ratio = np.zeros((B, K, hn_total), dtype=np.float32) if debug else None
    rc = lib().orc_estimate_voting_distribution(_p(mask, _i64p), _p(vertex, _f32p), _p(mean, _f32p),
                                                B, H, W, K, hn_total, ctypes.c_float(inlier_thresh),
                                                int(min_num), int(max_num), _p(idxs, _i32p), _p(selection, _f32p),
                                                ctypes.c_uint64(seed), int(img_base),
                                                _p(cov, _f32p), _p(hyp, _f32p), _p(ratio, _f32p))
    assert rc == 0
    if debug:
        return mean, cov, dict(hyp=hyp, ratio=ratio)
    return mean, cov
