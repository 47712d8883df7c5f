"""CPU tests of T-LESS's VSD layer (DESIGN.md 8f): the fp64 ray-casting oracle against closed forms, the numpy VSD
restatement against the reference's own vsd_utils (tests/golden/vsd.npz), the C ABI's argument validation, the Python
surface's errors, and the OpenGL drop-in on a miniature checkout."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import render_oracle
from vsd_cases import K_TLESS, box, vsd_restated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vsd.npz")


@pytest.fixture(scope="module")
def orc():
    render_oracle.build()
    return render_oracle


def _pose(t, R=None):
    p = np.zeros((3, 4))
    p[:, :3] = np.eye(3) if R is None else R
    p[:, 3] = t
    return p


def _quad(x0, x1, y0, y1, z0, z1=None):
    """Two triangles of the rectangle [x0,x1] x [y0,y1]; depth z0 at y0 and z1 at y1 (a tilted plane)."""
    z1 = z0 if z1 is None else z1
    v = np.array([[x0, y0, z0], [x1, y0, z0], [x1, y1, z1], [x0, y1, z1]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def test_oracle_plane_at_known_depth(orc):
    v, f = _quad(-4000, 4000, -4000, 4000, 500)
    o = orc.render_depth(v, f, _pose((0, 0, 0)), K_TLESS, (720, 540))
    assert np.all(np.abs(o["z"] - 500.0) <= 1e-9)


def test_oracle_cube_face_on_fixes_the_pixel_centres(orc):
    """A box centred on the optical axis: its silhouette is the front face, columns c with fx * X / Z + cx on either side
    of c + 0.5, rows likewise -- the (c + 0.5, r + 0.5) convention, not (c, r)."""
    v, f = box(60.0, 40.0, 50.0)
    Z = 700.0
    o = orc.render_depth(v, f, _pose((0, 0, Z)), K_TLESS, (720, 540))
    fx, cx, fy, cy = K_TLESS[0, 0], K_TLESS[0, 2], K_TLESS[1, 1], K_TLESS[1, 2]
    u = np.arange(720) + 0.5
    vv = np.arange(540) + 0.5
    cols = (u >= fx * -60 / (Z - 50) + cx) & (u <= fx * 60 / (Z - 50) + cx)
    rows = (vv >= fy * -40 / (Z - 50) + cy) & (vv <= fy * 40 / (Z - 50) + cy)
    assert np.array_equal(o["z"] > 0, rows[:, None] & cols[None, :])
    assert np.all(np.abs(o["z"][o["z"] > 0] - (Z - 50)) <= 1e-9)
    # the same box with the integer-coordinate convention would differ in at least one column here
    assert not np.array_equal(cols, ((u - 0.5) >= fx * -60 / (Z - 50) + cx) & ((u - 0.5) <= fx * 60 / (Z - 50) + cx))


def test_oracle_triangle_crossing_the_near_plane(orc):
    """A plane tilted from Z = -200 (top, behind the camera) to Z = 400 (bottom): pixels whose ray meets it in front of
    near are 0."""
    v, f = _quad(-300, 300, -300, 300, -200, 400)
    o = orc.render_depth(v, f, _pose((0, 0, 0)), K_TLESS, (720, 540), near=100, far=10000)
    fy, cy = K_TLESS[1, 1], K_TLESS[1, 2]
    # plane: Z = 100 + Y; the ray of row r has Y = yv * Z, yv = (r + 0.5 - cy) / fy
    yv = (np.arange(540) + 0.5 - cy) / fy
    zr = 100 / (1 - yv)
    z = o["z"]
    hit = z > 0
    assert hit.any() and (~hit).any()
    rows_hit = hit.any(axis=1)
    assert np.all(zr[rows_hit] >= 100 - 1e-6)
    for r in np.nonzero(rows_hit)[0]:
        assert np.allclose(z[r][hit[r]], zr[r], rtol=1e-12)
    assert np.all(~rows_hit[(zr < 100 - 1e-6) | (zr < 0)])


def test_oracle_mesh_behind_the_camera_and_beyond_far(orc):
    v, f = box()
    assert not orc.render_depth(v, f, _pose((0, 0, -700)), K_TLESS, (720, 540))["z"].any()
    assert not orc.render_depth(v, f, _pose((0, 0, 20000)), K_TLESS, (720, 540))["z"].any()
    assert orc.render_depth(v, f, _pose((0, 0, 20000)), K_TLESS, (720, 540), far=30000)["z"].any()


def test_vsd_restatement_equals_the_reference_bit_for_bit():
    g = np.load(GOLDEN)
    assert len(g["e"]) >= 16 and np.any(g["e"] == 1.0) and np.any(g["e"] < 0.3)
    for i in range(len(g["e"])):
        e = vsd_restated(g["depth_est"][i], g["depth_gt"][i], g["depth_test"][i], g["K"][i], int(g["delta"]),
                         int(g["tau"]))
        assert e == g["e"][i], (i, e, g["e"][i])


# ---- C ABI and Python surface, without a GPU --------------------------------------------------------------------------

def test_render_abi_validation(pvb):
    lib = pvb._lib.load()
    INV, WS = pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_ERR_WORKSPACE
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    rd = lambda *a: lib.pvb_render_depth(*a)   # noqa: E731
    ok = (p, 8, p, 12, p, 2, p, 0, p, 16, 16, 100.0, 10000.0)
    assert rd(*ok[:3], -1, *ok[4:], None, 0, None) == INV
    assert rd(*ok[:11], 0.0, 10000.0, None, 0, None) == INV                        # near must be > 0
    assert rd(*ok[:11], 100.0, 50.0, None, 0, None) == INV                         # far < near
    assert rd(*ok[:11], 100.0, float("inf"), None, 0, None) == INV
    assert rd(p, 8, None, 12, p, 2, p, 0, p, 16, 16, 100.0, 1e4, None, 0, None) == INV   # NULL faces
    assert rd(*ok[:7], -9, *ok[8:], None, 0, None) == INV                          # negative stride
    assert rd(*ok[:5], 70000, *ok[6:], None, 0, None) == INV
    assert rd(*ok, None, 0, None) == WS                                            # workspace missing
    need = lib.pvb_render_depth_workspace_bytes(2, 12)
    assert need >= 2 * 12 * 4 and lib.pvb_render_depth_workspace_bytes(0, 12) == 0
    assert rd(*ok, p + 1, need, None) == WS                                        # misaligned (or short)
    assert rd(*ok[:5], 0, *ok[6:], None, 0, None) == pvb._lib.PVB_OK               # n == 0: no-op
    assert len(lib.pvb_last_error()) > 0


def test_vsd_abi_validation(pvb):
    lib = pvb._lib.load()
    INV, WS = pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_ERR_WORKSPACE
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    v = lambda *a: lib.pvb_vsd(*a)   # noqa: E731
    ok = [p, 1, p, 2, 0, p, 2, 0, p, 3, p, 0, 8, 8, 15.0, 20.0, p]
    assert v(*ok, None, 0, None) == WS
    for i, bad in ((1, -1), (9, -1), (12, -8)):
        a = list(ok); a[i] = bad
        assert v(*a, None, 0, None) == INV
    a = list(ok); a[14] = float("nan")
    assert v(*a, None, 0, None) == INV
    a = list(ok); a[8] = None
    assert v(*a, None, 0, None) == INV
    a = list(ok); a[11] = -9
    assert v(*a, None, 0, None) == INV
    a = list(ok); a[9] = 0
    assert v(*a, None, 0, None) == pvb._lib.PVB_OK
    assert lib.pvb_vsd_workspace_bytes(3) >= 3 * 16 and lib.pvb_vsd_workspace_bytes(0) == 0


def test_python_errors_before_any_launch(pvb):
    v, f = box()
    with pytest.raises(RuntimeError, match="pts"):
        pvb.render_depth_batch(np.zeros((4, 2)), f, np.zeros((1, 3, 4)), K_TLESS, (64, 48))
    with pytest.raises(RuntimeError, match="poses"):
        pvb.render_depth_batch(v, f, np.zeros((1, 4, 4)), K_TLESS, (64, 48))
    with pytest.raises(RuntimeError, match="K"):
        pvb.render_depth_batch(v, f, np.zeros((2, 3, 4)), np.zeros((3, 3, 3)), (64, 48))
    with pytest.raises(RuntimeError, match="near"):
        pvb.render_depth_batch(v, f, np.zeros((1, 3, 4)), K_TLESS, (64, 48), near=0)
    with pytest.raises(RuntimeError, match="pairs"):
        pvb.vsd_batch(v, f, np.zeros((1, 3, 4)), np.zeros((1, 3, 4)), K_TLESS, np.zeros((1, 8, 8), np.float32),
                      np.zeros((2, 3)))
    assert pvb.render.vsd_batch is pvb.vsd_batch


def test_dropin_replaces_the_opengl_renderers(tmp_path):
    """A miniature checkout whose renderer modules import glumpy: after install_depth_renderer_as_reference(),
    vsd_utils' `from . import renderer` and icp_utils' `from lib.utils.renderer import opengl_utils` bind the twin and
    every other mode than depth raises NotImplementedError."""
    files = {
        "lib/__init__.py": "",
        "lib/utils/renderer/opengl_utils.py": "import glumpy\n",
        "lib/utils/vsd/renderer.py": "import glumpy\n",
        "lib/utils/vsd/misc.py": "MARK = 'real misc'\n",
        "lib/utils/vsd/visibility.py": "MARK = 'real visibility'\n",
        "lib/utils/vsd/vsd_utils.py": "import numpy as np\nfrom . import renderer, misc, visibility\n",
        "lib/utils/icp/icp_utils.py": "from lib.utils.renderer import opengl_utils\n",
    }
    for rel, text in files.items():
        q = tmp_path / rel
        q.parent.mkdir(parents=True, exist_ok=True)
        q.write_text(text)
    code = f"""
        import sys
        sys.path.insert(0, {str(tmp_path)!r})
        import clean_pvnet_b200 as pvb
        pvb.install_depth_renderer_as_reference()
        from lib.utils.vsd import vsd_utils
        from lib.utils.icp import icp_utils
        assert vsd_utils.renderer is pvb.render and icp_utils.opengl_utils is pvb.render
        assert vsd_utils.misc.MARK == 'real misc'
        import lib
        assert lib.__file__.startswith({str(tmp_path)!r})
        for call in (lambda: vsd_utils.renderer.render({{'pts': 0, 'faces': 0}}, (8, 8), None, None, None, mode='rgb'),
                     lambda: icp_utils.opengl_utils.NormalRender({{}}, (8, 8))):
            try:
                call()
                raise SystemExit('no NotImplementedError')
            except NotImplementedError:
                pass
        pvb.install_depth_renderer_as_reference()
        print('ok')
    """
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout
