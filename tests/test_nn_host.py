"""CPU tests of the nearest-neighbour port (lib/csrc/nn): the oracle's restatement of the reference predicate on known
answers, the C ABI's argument validation (before any CUDA call, so no device is needed), the Python surface, and the
opt-in drop-in on a miniature clean-pvnet checkout."""
import ctypes
import os
import subprocess
import sys
import textwrap
from fractions import Fraction

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def nn_oracle():
    import nn_oracle as mod
    mod.build()
    return mod


# A query and two points whose distances the reference's rounding orders one way and exact arithmetic the other:
# points (R1, R0) -- exact distance and plain fp32 (no fused multiply-add) pick index 0, the reference's
# fma(dz, dz, fma(dx, dx, RN(dy*dy))) picks index 1.
FMA_Q = np.array([1059139307, 1064876084, 1051350329], np.uint32).view(np.float32)
FMA_R0 = np.array([1051250303, 3201328162, 3203581360], np.uint32).view(np.float32)
FMA_R1 = np.array([1073124227, 1055130008, 3204237236], np.uint32).view(np.float32)


def _rn32(fr):
    """The fp32 nearest to the rational `fr` (ties to even)."""
    f = np.float32(float(fr))
    cands = (np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf)))
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - fr), int(c.view(np.uint32)) & 1))


def _pinned(r, q):
    """The reference's distance computed exactly in rationals, rounded where its PTX rounds."""
    fr = lambda v: Fraction(float(v))   # noqa: E731
    dx, dy, dz = (_rn32(fr(r[i]) - fr(q[i])) for i in range(3))
    d = _rn32(fr(dy) * fr(dy))
    d = _rn32(fr(dx) * fr(dx) + fr(d))
    return _rn32(fr(dz) * fr(dz) + fr(d))


def test_fma_rounding_decides_the_winner(nn_oracle):
    ref = np.stack([FMA_R1, FMA_R0])[None]
    que = FMA_Q[None, None]
    exact = ((ref[0].astype(np.float64) - que[0, 0].astype(np.float64)) ** 2).sum(-1)
    plain = np.array([np.float32(np.float32(d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) for d in ref[0] - que[0, 0]])
    assert exact.argmin() == 0 and plain.argmin() == 0
    assert _pinned(FMA_R0, FMA_Q) < _pinned(FMA_R1, FMA_Q)
    assert nn_oracle.nearest_point_idx(ref, que).tolist() == [[1]]


def test_duplicates_go_to_the_first_index(nn_oracle):
    ref = np.array([[[5, 5, 5], [1, 2, 3], [0, 0, 0], [1, 2, 3], [1, 2, 3]]], np.float32)
    que = np.array([[[1, 2, 3], [1.1, 2, 3], [0.4, 0.4, 0.4]]], np.float32)
    assert nn_oracle.nearest_point_idx(ref, que).tolist() == [[1, 1, 2]]
    assert nn_oracle.nearest_point_idx(ref[..., :2], que[..., :2]).tolist() == [[1, 1, 2]]


def test_exclude_self(nn_oracle):
    pts = np.array([[[0, 0], [0, 0], [3, 0], [3.5, 0], [10, 10]]], np.float32)
    assert nn_oracle.nearest_point_idx(pts, pts).tolist() == [[0, 0, 2, 3, 4]]
    assert nn_oracle.nearest_point_idx(pts, pts, exclude_self=True).tolist() == [[1, 0, 3, 2, 3]]
    one = np.zeros((1, 1, 3), np.float32)
    assert nn_oracle.nearest_point_idx(one, one, exclude_self=True).tolist() == [[0]]   # no candidate: index 0


def test_nan_inf_and_flt_max_never_win(nn_oracle):
    nan, inf, big = np.float32("nan"), np.float32("inf"), np.float32(1e30)
    ref = np.array([[[nan, 0, 0], [inf, 0, 0], [big, 0, 0], [3, 0, 0], [nan, nan, nan]]], np.float32)
    que = np.array([[[0, 0, 0], [nan, 0, 0], [-inf, 0, 0], [2, 0, 0]]], np.float32)
    # (big)^2 overflows to inf; a NaN query has no finite distance; -inf - 3 = -inf -> inf
    assert nn_oracle.nearest_point_idx(ref, que).tolist() == [[3, 0, 0, 3]]
    # fma(x, x, RN(y*y)) with x = 2^64 - 2^40 rounds to exactly FLT_MAX for y = 2^52 (not < FLT_MAX: index 0 stays),
    # and to the float below it for y = 2^51 (taken)
    x = 2.0 ** 64 - 2.0 ** 40
    zero = np.zeros((1, 1, 2), np.float32)
    assert nn_oracle.nearest_point_idx(np.array([[[nan, 0], [x, 2.0 ** 52]]], np.float32), zero).tolist() == [[0]]
    assert nn_oracle.nearest_point_idx(np.array([[[nan, 0], [x, 2.0 ** 51]]], np.float32), zero).tolist() == [[1]]


@pytest.mark.parametrize("dim", [2, 3])
def test_oracle_matches_float64_argmin_on_tie_free_data(nn_oracle, dim):
    rng = np.random.default_rng(dim)
    ref = rng.random((3, 400, dim)).astype(np.float32)
    que = rng.random((3, 300, dim)).astype(np.float32)
    d = ((ref[:, None].astype(np.float64) - que[:, :, None].astype(np.float64)) ** 2).sum(-1)
    srt = np.sort(d, -1)
    assert (srt[..., 1] - srt[..., 0] > 1e-6 * srt[..., 1]).all()        # well separated: no near-ties
    assert np.array_equal(nn_oracle.nearest_point_idx(ref, que), d.argmin(-1))


# ---- C ABI ------------------------------------------------------------------------------------------------------------

def test_nearest_point_validation(pvb):
    lib = pvb._lib.load()
    INV, WS = pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_ERR_WORKSPACE
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    nn = lib.pvb_nearest_point_idx
    assert nn(p, p, p, -1, 4, 4, 3, 0, None, 0, None) == INV
    assert nn(p, p, p, 1, -4, 4, 3, 0, None, 0, None) == INV
    assert nn(p, p, p, 1, 4, -4, 3, 0, None, 0, None) == INV
    for dim in (0, 1, 4):
        assert nn(p, p, p, 1, 4, 4, dim, 0, None, 0, None) == INV
        assert b"dim" in lib.pvb_last_error()
    assert nn(None, p, p, 1, 4, 4, 3, 0, None, 0, None) == INV
    assert nn(p, None, p, 1, 4, 4, 2, 0, None, 0, None) == INV
    assert nn(p, p, None, 1, 4, 4, 2, 0, None, 0, None) == INV
    # empty problems are a no-op, whatever the pointers
    assert nn(None, None, None, 0, 4, 4, 3, 0, None, 0, None) == pvb._lib.PVB_OK
    assert nn(None, None, None, 2, 4, 0, 3, 0, None, 0, None) == pvb._lib.PVB_OK
    # one image of 20000 points cannot fill the GPU: the split path needs a merge key per query
    need = lib.pvb_nearest_point_workspace_bytes(1, 20000, 20000)
    assert need == 20000 * 8
    assert nn(p, p, p, 1, 20000, 20000, 3, 0, None, 0, None) == WS
    assert nn(p, p, p, 1, 20000, 20000, 3, 0, p, need - 1, None) == WS
    assert b"workspace" in lib.pvb_last_error()
    # shapes that fill the GPU in one pass, or too few reference points to split, need none
    assert lib.pvb_nearest_point_workspace_bytes(16, 700, 102400) == 0
    assert lib.pvb_nearest_point_workspace_bytes(3, 60, 20000) == 0
    assert lib.pvb_nearest_point_workspace_bytes(-1, 10, 10) == 0


def test_add_metric_validation(pvb):
    lib = pvb._lib.load()
    INV, WS = pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_ERR_WORKSPACE
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    am = lib.pvb_add_metric
    assert am(p, p, p, p, -1, 10, 1, p, 4096, None) == INV
    assert am(p, p, p, p, 1, -10, 1, p, 4096, None) == INV
    assert am(p, p, p, p, 1, 10, 2, p, 4096, None) == INV
    assert am(None, p, p, p, 1, 10, 0, p, 4096, None) == INV
    assert am(p, None, p, p, 1, 10, 0, p, 4096, None) == INV
    assert am(p, p, None, p, 1, 10, 0, p, 4096, None) == INV
    assert am(p, p, p, None, 1, 10, 0, p, 4096, None) == INV
    assert am(None, None, None, None, 0, 10, 1, None, 0, None) == pvb._lib.PVB_OK
    for syn in (0, 1):
        need = lib.pvb_add_metric_workspace_bytes(4, 5000, syn)
        assert need >= 4 * 8
        assert am(p, p, p, p, 4, 5000, syn, None, 0, None) == WS
        assert am(p, p, p, p, 4, 5000, syn, p, need - 1, None) == WS
    # ADD-S split over pn needs the merge keys, ADD only the per-CTA partial sums
    assert lib.pvb_add_metric_workspace_bytes(4, 5000, 1) > 4 * 5000 * 8 > lib.pvb_add_metric_workspace_bytes(4, 5000, 0)


def test_python_surface_rejects_bad_inputs(pvb):
    with pytest.raises(AssertionError):                       # nn_utils.py:6
        pvb.find_nearest_point_idx(np.zeros((4, 1)), np.zeros((4, 1)))
    with pytest.raises(AssertionError):
        pvb.find_nearest_point_idx(np.zeros((4, 3)), np.zeros((4, 2)))
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        pvb.nearest_point_idx(torch.zeros(1, 4, 3), torch.zeros(1, 4, 3))
    assert pvb.nn.find_nearest_point_idx is pvb.find_nearest_point_idx


# ---- drop-in ----------------------------------------------------------------------------------------------------------

def _run(code, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=cwd, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    return r.stdout


def _checkout(tmp_path):
    """A miniature clean-pvnet tree whose lib/csrc/nn (a namespace package, as in the reference) has the real nn_utils,
    which imports the cffi extension -- never built here -- and both evaluators importing it at module level."""
    files = {
        "lib/__init__.py": "",
        "lib/config/__init__.py": "cfg = 'real lib.config'\n",
        "lib/csrc/nn/nn_utils.py": "from lib.csrc.nn._ext import lib, ffi\n",
        "lib/csrc/nn/_ext.py": "raise RuntimeError('cffi extension imported')\n",
        "lib/evaluators/__init__.py": "",
        "lib/evaluators/linemod/__init__.py": "",
        "lib/evaluators/linemod/pvnet.py": "from lib.config import cfg\nfrom lib.csrc.nn import nn_utils\n",
        "lib/evaluators/tless_test/__init__.py": "",
        "lib/evaluators/tless_test/pvnet.py": "from lib.csrc.nn import nn_utils\n",
    }
    for rel, text in files.items():
        f = tmp_path / rel
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(text)
    return str(tmp_path)


def test_install_nn_binds_the_twin_without_the_cffi_extension(tmp_path):
    tree = _checkout(tmp_path)
    code = f"""
        import sys
        sys.path.insert(0, {tree!r})
        import clean_pvnet_b200
        clean_pvnet_b200.install_nn_as_reference_module()
        from lib.csrc.nn import nn_utils
        assert nn_utils is clean_pvnet_b200.nn
        assert nn_utils.find_nearest_point_idx is clean_pvnet_b200.find_nearest_point_idx
        from lib.evaluators.linemod import pvnet as linemod
        from lib.evaluators.tless_test import pvnet as tless
        assert linemod.nn_utils is nn_utils and tless.nn_utils is nn_utils and linemod.cfg == 'real lib.config'
        import lib, lib.csrc
        assert lib.__file__.startswith({tree!r}) and not getattr(lib, '__pvb_stand_in__', False)
        assert not getattr(lib.csrc, '__pvb_stand_in__', False)
        assert 'lib.csrc.nn._ext' not in sys.modules
        clean_pvnet_b200.install_as_reference_module()       # the voting-layer drop-in leaves the twin in place
        clean_pvnet_b200.install_nn_as_reference_module()    # idempotent
        from lib.csrc.nn import nn_utils as again
        assert again is clean_pvnet_b200.nn and 'lib.csrc.nn._ext' not in sys.modules
        print('ok')
    """
    assert "ok" in _run(code, cwd=tree)


def test_install_nn_without_a_checkout_uses_stand_ins(tmp_path):
    code = """
        import clean_pvnet_b200
        clean_pvnet_b200.install_nn_as_reference_module()
        from lib.csrc.nn.nn_utils import find_nearest_point_idx
        import lib
        assert lib.__pvb_stand_in__ and find_nearest_point_idx is clean_pvnet_b200.find_nearest_point_idx
        print('ok')
    """
    assert "ok" in _run(code, cwd=str(tmp_path))
