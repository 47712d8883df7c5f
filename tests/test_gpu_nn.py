"""The nearest-neighbour kernels (csrc/nn.cu) against the reference's own kernel (oracle/_ref/libnn_ref.so, built
unmodified by oracle/build_nn_ref.py; those comparisons skip only where it was not built) and the C oracle: indices
bit-equal on every shape, on near-ties, duplicates, NaN and inf, on the single-pass and the split-and-merge path; and the
batched ADD / ADD-S distance against the evaluator's own formulas."""
import ctypes
import os

import numpy as np
import pytest
import torch

from test_nn_host import FMA_Q, FMA_R0, FMA_R1

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def nn_oracle():
    import nn_oracle as mod
    mod.build()
    return mod


REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libnn_ref.so")
_REF = []


def _ref_lib():
    if not os.path.exists(REF_LIB):
        return None
    if not _REF:
        lib = ctypes.CDLL(REF_LIB)
        f = lib.findNearestPointIdxLauncher
        f.restype = None
        f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5
        _REF.append(lib)
    return _REF[0]


def ref_nearest(ref, que, exclude_self=False):
    """The reference launcher on host arrays, as nn_utils.py:10-18 calls it (b, exclude_self generalised)."""
    lib = _ref_lib()
    ref = np.ascontiguousarray(ref, np.float32)
    que = np.ascontiguousarray(que, np.float32)
    b, pn1, dim = ref.shape
    idxs = np.zeros((b, que.shape[1]), np.int32)
    lib.findNearestPointIdxLauncher(ref.ctypes.data, que.ctypes.data, idxs.ctypes.data, b, pn1, que.shape[1], dim,
                                    int(exclude_self))
    return idxs


def _cloud(rng, kind, b, n, dim):
    if kind == "uniform":
        return rng.random((b, n, dim)).astype(np.float32)
    if kind == "clustered":            # a coarse lattice: many equal and near-equal distances
        c = rng.integers(0, 6, size=(b, n, dim)).astype(np.float32) * np.float32(0.25)
        return c + (rng.integers(0, 3, size=(b, n, dim)) * np.float32(1e-7)).astype(np.float32)
    if kind == "tiny":                 # squares in the subnormal range: the kernels must not flush them
        return (rng.random((b, n, dim)) * 1e-20).astype(np.float32)
    if kind == "special":              # duplicates, NaN, +-inf, huge values
        c = rng.random((b, n, dim)).astype(np.float32)
        if n > 1:
            c[:, 1::3] = c[:, 0:1]
        m = rng.random((b, n, dim))
        c[m < 0.05] = np.nan
        c[(m >= 0.05) & (m < 0.08)] = np.inf
        c[(m >= 0.08) & (m < 0.10)] = -np.inf
        c[(m >= 0.10) & (m < 0.12)] = np.float32(3e19)
        return c
    raise ValueError(kind)


def _check(pvb, nn_oracle, ref, que, exclude_self=False, reference=True):
    got = pvb.nearest_point_idx(torch.from_numpy(ref).cuda(), torch.from_numpy(que).cuda(), exclude_self).cpu().numpy()
    assert got.dtype == np.int32
    want = nn_oracle.nearest_point_idx(ref, que, exclude_self)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    if reference and _ref_lib() is not None:
        assert np.array_equal(got, ref_nearest(ref, que, exclude_self))
    return got


# (b, pn1, pn2, dim, exclude_self, kind); workspace bytes > 0 <=> the split-and-merge path
CASES = [
    (1, 1, 1, 3, False, "uniform"),
    (1, 7, 1000, 2, False, "uniform"),
    (1, 20000, 20000, 3, False, "uniform"),        # split
    (1, 5000, 3000, 2, True, "uniform"),           # split
    (3, 4000, 4000, 3, True, "clustered"),         # split, ref is que
    (3, 1300, 900, 2, False, "clustered"),
    (3, 60, 20000, 3, False, "clustered"),         # pn1 too short to split: single pass
    (16, 2500, 1200, 3, False, "special"),         # split
    (16, 600, 333, 2, False, "special"),
    (16, 700, 102400, 3, False, "uniform"),        # fills the GPU: single pass
    (16, 1000, 2000, 3, False, "tiny"),
]


@pytest.mark.parametrize("b,pn1,pn2,dim,excl,kind", CASES)
def test_indices_bit_equal_to_reference_and_oracle(pvb, nn_oracle, b, pn1, pn2, dim, excl, kind):
    rng = np.random.default_rng(b * 7919 + pn1 * 31 + pn2 + dim)
    ref = _cloud(rng, kind, b, pn1, dim)
    que = ref.copy() if excl and pn1 == pn2 else _cloud(rng, kind, b, pn2, dim)
    if kind == "clustered" and pn2 <= pn1:
        que[:, : pn2 // 2] = ref[:, : pn2 // 2]                 # exact hits next to lattice ties
    _check(pvb, nn_oracle, ref, que, excl)


def test_both_paths_are_exercised(pvb):
    ws = pvb._lib.load().pvb_nearest_point_workspace_bytes
    split = [c for c in CASES if ws(c[0], c[1], c[2]) > 0]
    single = [c for c in CASES if ws(c[0], c[1], c[2]) == 0]
    assert len(split) >= 4 and len(single) >= 4
    assert any(c[2] > 20000 for c in single) and any(c[1] >= 20000 for c in split)


def test_fma_rounding_case_and_empty_reference(pvb, nn_oracle):
    ref = np.stack([FMA_R1, FMA_R0])[None]
    assert _check(pvb, nn_oracle, ref, FMA_Q[None, None]).tolist() == [[1]]
    # no reference point at all: every query gets index 0, like the reference's untouched min_idx
    got = pvb.nearest_point_idx(torch.zeros(2, 0, 3, device="cuda"), torch.rand(2, 5, 3, device="cuda"))
    assert got.tolist() == [[0] * 5] * 2


def test_find_nearest_point_idx_is_nn_utils(pvb, nn_oracle):
    """The numpy entry on what the evaluator passes (float64 model clouds), against nn_utils.py:5-20's recipe."""
    rng = np.random.default_rng(5)
    for pn1, pn2, dim in [(20000, 20000, 3), (1000, 5000, 3), (640, 480, 2)]:
        ref_pts = rng.normal(size=(pn1, dim)) * 0.1
        que_pts = ref_pts[rng.integers(0, pn1, pn2)] + rng.normal(size=(pn2, dim)) * 1e-3
        got = pvb.find_nearest_point_idx(ref_pts, que_pts)
        assert got.dtype == np.int32 and got.shape == (pn2,)
        r32 = np.ascontiguousarray(ref_pts[None], np.float32)
        q32 = np.ascontiguousarray(que_pts[None], np.float32)
        want = ref_nearest(r32, q32)[0] if _ref_lib() is not None else nn_oracle.nearest_point_idx(r32, q32)[0]
        assert np.array_equal(got, want)


def _rot(rng, n, scale=np.pi):
    aa = rng.normal(size=(n, 3))
    aa *= (rng.random((n, 1)) * scale) / np.linalg.norm(aa, axis=1, keepdims=True)
    out = []
    for w in aa:
        t = np.linalg.norm(w)
        k = w / t
        K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        out.append(np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K)
    return np.stack(out)


def _poses(rng, n, pn):
    model = (rng.normal(size=(pn, 3)) * [0.05, 0.03, 0.04]).astype(np.float32)   # a LINEMOD-sized object, metres
    gt = np.concatenate([_rot(rng, n), (rng.normal(size=(n, 3, 1)) * 0.1 + [[0], [0], [1.0]])], 2)
    pred = gt.copy()
    # half the pairs close (well inside 0.1 * diameter), half clearly off (well outside)
    off = np.where(np.arange(n)[:, None, None] % 2 == 0, 1e-3, 0.3)
    pred[:, :, :3] = _rot(rng, n, 0.02) @ gt[:, :, :3]
    pred[:, :, 3:] += rng.normal(size=(n, 3, 1)) * off
    return model, pred, gt


def _evaluator_mean(model, pose_pred, pose_targets, syn, nearest):
    """Evaluator.add_metric (lib/evaluators/linemod/pvnet.py:68-82), up to the threshold."""
    model_pred = np.dot(model, pose_pred[:, :3].T) + pose_pred[:, 3]
    model_targets = np.dot(model, pose_targets[:, :3].T) + pose_targets[:, 3]
    if syn:
        idxs = nearest(model_pred, model_targets)
        return np.mean(np.linalg.norm(model_pred[idxs] - model_targets, 2, 1))
    return np.mean(np.linalg.norm(model_pred - model_targets, axis=-1))


@pytest.mark.parametrize("n,pn", [(1, 5000), (5, 2000), (3, 20000), (800, 1000)])
def test_add_metric_batch_matches_the_evaluator(pvb, nn_oracle, n, pn):
    rng = np.random.default_rng(n * 100003 + pn)
    model, pred, gt = _poses(rng, n, pn)
    diameter = float(np.max(np.linalg.norm(model[:, None] - model[None, :200], axis=-1)))

    def nearest(a, b):
        a32, b32 = np.ascontiguousarray(a[None], np.float32), np.ascontiguousarray(b[None], np.float32)
        return ref_nearest(a32, b32)[0] if _ref_lib() is not None else nn_oracle.nearest_point_idx(a32, b32)[0]

    for syn in (False, True):
        got = pvb.add_metric_batch(torch.from_numpy(model).cuda(), torch.from_numpy(pred).cuda(),
                                   torch.from_numpy(gt).cuda(), syn)
        assert got.dtype == torch.float64 and got.shape == (n,)
        got = got.cpu().numpy()
        check = range(n) if n <= 8 else rng.choice(n, 8, replace=False)
        for i in check:
            want = _evaluator_mean(model.astype(np.float64), pred[i], gt[i], syn, nearest)
            assert np.isclose(got[i], want, rtol=1e-9, atol=0), (i, got[i], want)
            assert abs(want - 0.1 * diameter) > 0.05 * diameter            # away from the threshold
            assert (got[i] < 0.1 * diameter) == (want < 0.1 * diameter)
    ws = pvb._lib.load().pvb_add_metric_workspace_bytes
    assert (ws(n, pn, 1) > ws(n, pn, 0)) == (n * ((pn + 2047) // 2048) < 792)   # split ADD-S keeps merge keys


def test_add_metric_all_pairs_like_adi_metric(pvb):
    """T-LESS's adi_metric: every (prediction, ground truth) pair, expanded into rows by the caller."""
    rng = np.random.default_rng(11)
    model, pred, gt = _poses(rng, 6, 3000)
    pp = np.repeat(pred[:3], 3, axis=0)
    gg = np.tile(gt[3:], (3, 1, 1))
    rows = pvb.add_metric_batch(model, torch.from_numpy(pp).cuda(), torch.from_numpy(gg).cuda(), True).cpu().numpy()
    for i in range(3):
        for j in range(3):
            one = pvb.add_metric_batch(model, torch.from_numpy(pred[i:i + 1]).cuda(),
                                       torch.from_numpy(gt[3 + j:4 + j]).cuda(), True).cpu().numpy()
            assert rows[i * 3 + j] == one[0]
