"""CPU tests of the farthest-point-sampling port (lib/csrc/fps): the fixture against the reference build and the numpy
restatement, the C ABI's argument validation (before any CUDA call, so no device is needed), the Python surface, and the
opt-in drop-in on a miniature clean-pvnet checkout."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import fps_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_restatement_matches_the_fixture():
    for kind, pn, sn, seed, init_center, start, idxs in fps_cases.load_golden():
        got = fps_cases.fps_restated(fps_cases.cloud(kind, pn, seed), sn, None if init_center else start)
        assert np.array_equal(got, idxs), (kind, pn, sn, init_center)


def test_fixture_covers_the_reference_corner_cases():
    g = fps_cases.load_golden()
    same = [c for c in g if c[0] == "same" and c[4]]
    assert same and all(not c[6].any() for c in same)                     # all-identical clouds give [0, 0, ...]
    over = [c for c in g if c[2] > c[1] > 1]
    assert over and all((c[6][c[1]:] == 0).all() for c in over)          # sn > pn repeats index 0
    assert {c[1] for c in g} >= set(fps_cases.BOUNDARY_PN) | {1, 2, 31, 32, 33, 1000, 100000, 1000000}
    assert {c[2] for c in g if c[1] == 1000} >= {0, 1, 8, 64, 1000, 1003}


def test_fixture_equals_the_reference_build():
    lib = fps_cases.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libfps_ref.so not built (no reference checkout)")
    for kind, pn, sn, seed, init_center, start, idxs in fps_cases.load_golden():
        pts = fps_cases.cloud(kind, pn, seed)
        if init_center:
            assert np.array_equal(fps_cases.ref_fps(lib, pts, sn, 1), idxs), (kind, pn, sn)
        elif sn and pn <= 100000:
            # the reference draws its own start; from that start it must equal the restatement the fixture equals
            r = fps_cases.ref_fps(lib, pts, sn, 0)
            assert np.array_equal(r, fps_cases.fps_restated(pts, sn, int(r[0]))), (kind, pn, sn)


def test_fps_validation(pvb):
    lib = pvb._lib.load()
    OK, INV, WS = pvb._lib.PVB_OK, pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_ERR_WORKSPACE
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    cnt = np.array([10, 7], np.int32)
    st = np.array([0, 6], np.int32)
    c, s = cnt.ctypes.data, st.ctypes.data
    need = lib.pvb_fps_workspace_bytes(2, 10)
    assert need >= 2 * 2 * 4
    fps = lib.pvb_farthest_point_sampling
    for ic in (0, 1):
        assert fps(p, c, s, ic, p, -1, 10, 8, p, need, None) == INV
        assert fps(p, c, s, ic, p, 2, -10, 8, p, need, None) == INV
        assert fps(p, c, s, ic, p, 2, 10, -8, p, need, None) == INV
        assert fps(None, c, s, ic, p, 2, 10, 8, p, need, None) == INV
        assert fps(p, None, s, ic, p, 2, 10, 8, p, need, None) == INV
        assert fps(p, c, s, ic, None, 2, 10, 8, p, need, None) == INV
        for bad in ([0, 7], [11, 7], [10, -1]):
            assert fps(p, np.array(bad, np.int32).ctypes.data, s, ic, p, 2, 10, 8, p, need, None) == INV
            assert b"points" in lib.pvb_last_error()
        assert fps(p, c, s, ic, p, 2, 10, 8, None, 0, None) == WS
        assert fps(p, c, s, ic, p, 2, 10, 8, p, need - 1, None) == WS
        assert b"workspace" in lib.pvb_last_error()
        # empty problems are a no-op, whatever the pointers
        assert fps(None, None, None, ic, None, 0, 10, 8, None, 0, None) == OK
        assert fps(None, None, None, ic, None, 2, 10, 0, None, 0, None) == OK
    # the random mode needs its starts, each inside its cloud; init_center ignores them
    assert fps(p, c, None, 0, p, 2, 10, 8, p, need, None) == INV
    for bad in ([10, 6], [0, 7], [-1, 0]):
        assert fps(p, c, np.array(bad, np.int32).ctypes.data, 0, p, 2, 10, 8, p, need, None) == INV
        assert b"starts" in lib.pvb_last_error()
    # every cloud of n <= 8192 points fits one CTA: only the tables; beyond, the streamed min_dist of each cloud
    assert lib.pvb_fps_workspace_bytes(2, 8192) == 256
    assert lib.pvb_fps_workspace_bytes(3, 10000) == 256 + 3 * (10000 - 8192) * 4
    assert lib.pvb_fps_workspace_bytes(0, 10) == 0 and lib.pvb_fps_workspace_bytes(-1, 10) == 0


def test_python_surface_rejects_bad_inputs(pvb):
    with pytest.raises(AssertionError):                       # fps_utils.py:7
        pvb.farthest_point_sampling(np.zeros((4, 2)), 2)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        pvb.farthest_point_sampling_batch(torch.zeros(1, 4, 3), 2)
    assert pvb.fps.farthest_point_sampling is pvb.farthest_point_sampling


# ---- drop-in ----------------------------------------------------------------------------------------------------------

def _run(code, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=cwd, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    return r.stdout


def _checkout(tmp_path):
    """A miniature clean-pvnet tree whose lib/csrc/fps (a namespace package, as in the reference) has the real fps_utils,
    which imports the cffi extension -- never built here -- and tools/handle_custom_dataset importing it at module
    level."""
    files = {
        "lib/__init__.py": "",
        "lib/config/__init__.py": "cfg = 'real lib.config'\n",
        "lib/csrc/fps/fps_utils.py": "from lib.csrc.fps._ext import lib, ffi\n",
        "lib/csrc/fps/_ext.py": "raise RuntimeError('cffi extension imported')\n",
        "lib/utils/__init__.py": "",
        "lib/utils/base_utils.py": "real = True\n",
        "tools/__init__.py": "",
        "tools/handle_custom_dataset.py": "from lib.csrc.fps import fps_utils\nfrom lib.utils import base_utils\n"
                                          "def sample_fps_points(pts):\n"
                                          "    return fps_utils.farthest_point_sampling(pts, 8, True)\n",
    }
    for rel, text in files.items():
        f = tmp_path / rel
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(text)
    return str(tmp_path)


def test_install_fps_binds_the_twin_without_the_cffi_extension(tmp_path):
    tree = _checkout(tmp_path)
    code = f"""
        import sys
        sys.path.insert(0, {tree!r})
        import clean_pvnet_b200
        clean_pvnet_b200.install_fps_as_reference_module()
        from lib.csrc.fps import fps_utils
        assert fps_utils is clean_pvnet_b200.fps
        assert fps_utils.farthest_point_sampling is clean_pvnet_b200.farthest_point_sampling
        from tools import handle_custom_dataset as h
        assert h.fps_utils is fps_utils and h.base_utils.real
        import lib, lib.csrc, lib.config
        assert lib.__file__.startswith({tree!r}) and not getattr(lib, '__pvb_stand_in__', False)
        assert not getattr(lib.csrc, '__pvb_stand_in__', False) and lib.config.cfg == 'real lib.config'
        assert 'lib.csrc.fps._ext' not in sys.modules
        clean_pvnet_b200.install_nn_as_reference_module()    # the other drop-ins leave the twin in place
        clean_pvnet_b200.install_fps_as_reference_module()   # idempotent
        from lib.csrc.fps import fps_utils as again
        assert again is clean_pvnet_b200.fps and 'lib.csrc.fps._ext' not in sys.modules
        print('ok')
    """
    assert "ok" in _run(code, cwd=tree)


def test_install_fps_without_a_checkout_uses_stand_ins(tmp_path):
    code = """
        import clean_pvnet_b200
        clean_pvnet_b200.install_fps_as_reference_module()
        from lib.csrc.fps.fps_utils import farthest_point_sampling
        import lib
        assert lib.__pvb_stand_in__ and farthest_point_sampling is clean_pvnet_b200.farthest_point_sampling
        print('ok')
    """
    assert "ok" in _run(code, cwd=str(tmp_path))
