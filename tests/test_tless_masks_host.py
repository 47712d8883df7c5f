"""CPU tests of T-LESS's instance masks (DESIGN.md 8k): the numpy restatement against the reference's own
handle_test_data code (tests/golden/tless_masks.npz), the C ABI's argument validation, the Python surface's errors, and
the OpenGL drop-in on a miniature checkout."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tless_mask_cases import compose_restated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "tless_masks.npz")


def golden_cases():
    g = np.load(GOLDEN)
    return [{k: g[f"c{i}_{k}"] for k in ("name", "depth", "obj_ids", "label", "a_pixel_num", "pixel_num", "bbox", "area")}
            for i in range(int(g["n_cases"]))]


def test_fixture_covers_the_cases_the_semantics_turn_on():
    cs = {str(c["name"]): c for c in golden_cases()}
    assert {c["depth"].shape[0] for c in cs.values()} >= {1, 20}
    assert any(c["depth"].shape[1:] == (540, 720) for c in cs.values())
    assert any(c["depth"].shape[1] % 32 and c["depth"].shape[2] % 32 for c in cs.values())
    far = cs["far_plane"]                                    # 10000 mm: rendered, never labelled
    assert far["a_pixel_num"][0] == far["depth"].shape[1] * far["depth"].shape[2] and far["pixel_num"][0] == 0
    occ = cs["occluded_and_empty"]
    assert occ["a_pixel_num"][1] > 0 and occ["pixel_num"][1] == 0 and occ["a_pixel_num"][2] == 0
    assert tuple(occ["bbox"][2]) == (0, 0, 0, 0)
    d = cs["same_key"]["depth"]
    assert len(np.unique(d[d != 0])) == 2 and len(np.unique(d[d != 0] / np.float32(1000))) == 1


def test_restatement_equals_the_reference_bit_for_bit():
    for c in golden_cases():
        label, a, p, box = compose_restated(c["depth"], c["obj_ids"])
        name = str(c["name"])
        assert label.dtype == c["label"].dtype and np.array_equal(label, c["label"]), name
        assert np.array_equal(a, c["a_pixel_num"]), name
        assert np.array_equal(p, c["pixel_num"]) and np.array_equal(p, c["area"]), name
        assert np.array_equal(box, c["bbox"]), name


# ---- C ABI and Python surface, without a GPU --------------------------------------------------------------------------

def _i32(*v):
    a = np.array(v, np.int32)
    return a, a.ctypes.data_as(ctypes.c_void_p)


def test_instance_masks_abi_validation(pvb):
    lib = pvb._lib.load()
    OK, INV, WS = pvb._lib.PVB_OK, pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_ERR_WORKSPACE
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    keep = []

    def call(slot=(0, 1, 0), obj=(3, 3, 30), first=(0, 2, 3), B=2, n_depth=2, H=8, W=8, ws=None, ws_bytes=0, n=None,
             depth=p):
        s, obj_, f = _i32(*slot), _i32(*obj), _i32(*first)
        keep.extend((s, obj_, f))
        return lib.pvb_instance_masks(depth, n_depth, s[1], obj_[1], len(obj) if n is None else n, f[1], B, H, W, p, p, p,
                                      p, ws, ws_bytes, None)

    assert call() == WS                                                   # workspace missing
    need = lib.pvb_instance_masks_workspace_bytes(2, 3)
    assert need >= 3 * 24 and lib.pvb_instance_masks_workspace_bytes(0, 3) == 0
    assert call(ws=p + 1, ws_bytes=need) == WS                            # misaligned
    assert call(obj=(3, 3, 33)) == INV                                    # 33 * 1000 + 0 > 32767
    assert call(obj=(-33, 3, 30)) == INV                                  # below -32768
    assert call(first=(0, 0, 3)) == INV                                   # an empty range
    assert call(first=(0, 2, 4)) == INV                                   # past n
    assert call(first=(-1, 2, 3)) == INV
    assert call(first=(2, 1, 3)) == INV                                   # decreasing
    assert call(slot=(0, 2, 0)) == INV                                    # slot outside [0, n_depth)
    assert call(slot=(0, -1, 0)) == INV
    assert call(H=1 << 16, W=1 << 15) == INV                              # H * W >= 2^31
    assert call(B=-1) == INV and call(H=-1) == INV
    assert call(B=70000) == INV
    assert call(depth=None) == INV
    assert call(B=0) == OK                                                # no-op
    assert len(lib.pvb_last_error()) > 0
    # obj_id 32: instance_id 767 gives 32767, the last label int16 holds; 768 gives 32768
    assert call(slot=[0] * 769, obj=[32] * 769, first=(0, 768, 769), n_depth=1) == WS
    assert call(slot=[0] * 769, obj=[32] * 769, first=(0, 769), B=1, n_depth=1) == INV
    many = 2049
    assert call(slot=[0] * many, obj=[0] * many, first=(0, many), B=1, n_depth=1) == INV     # > 2048 per image


def test_python_errors_before_any_launch(pvb):
    d = np.zeros((2, 8, 8), np.float32)
    with pytest.raises(RuntimeError, match="non-decreasing"):
        pvb.instance_masks_from_depth(d, [0, 1], [1, 1], [1, 0])
    with pytest.raises(RuntimeError, match="int16"):
        pvb.instance_masks_from_depth(d, [0, 1], [1, 33], [0, 0])
    with pytest.raises(RuntimeError, match="slot"):
        pvb.instance_masks_from_depth(d, [0, 2], [1, 1], [0, 0])
    with pytest.raises(RuntimeError, match="depth"):
        pvb.instance_masks_from_depth(d[0], [0], [1], [0])
    mesh = (np.zeros((3, 3), np.float32), np.array([[0, 1, 2]], np.int32))
    poses = np.zeros((2, 3, 4))
    with pytest.raises(RuntimeError, match="mesh_index"):
        pvb.instance_masks_batch([mesh], [0, 1], [1, 1], [0, 0], poses, np.eye(3), (8, 8))
    with pytest.raises(RuntimeError, match="poses"):
        pvb.instance_masks_batch([mesh], [0, 0], [1, 1], [0, 0], poses[:1], np.eye(3), (8, 8))
    with pytest.raises(RuntimeError, match="K"):
        pvb.instance_masks_batch([mesh], [0, 0], [1, 1], [0, 0], poses, np.zeros((2, 3)), (8, 8))
    with pytest.raises(RuntimeError, match="image_index"):
        pvb.instance_masks_batch([mesh], [0, 0], [1, 1], [0, 2], poses, np.zeros((2, 3, 3)), (8, 8))
    with pytest.raises(RuntimeError, match="near"):
        pvb.instance_masks_batch([mesh], [0, 0], [1, 1], [0, 0], poses, np.eye(3), (8, 8), near=0)
    assert pvb.render.instance_masks_batch is pvb.instance_masks_batch


TLESS_FILES = {
    # the imports of lib/datasets/tless/opengl_renderer.py, handle_test_data.py and handle_ag_data.py, over a backend
    # that needs glumpy
    "lib/__init__.py": "",
    "lib/datasets/__init__.py": "MARK = 'real datasets'\n",
    "lib/datasets/tless/opengl_backend.py": "import glumpy\n",
    "lib/datasets/tless/opengl_renderer.py":
        "import numpy as np\nfrom lib.datasets.tless import opengl_backend\n\n\n"
        "def render(model, pose, K, w, h, render_type='depth'):\n"
        "    depth = opengl_backend.render(model, im_size=[w, h], K=K, R=pose[:, :3], t=pose[:, 3:] * 1000.,\n"
        "                                  clip_near=10, clip_far=10000, mode='depth')\n"
        "    return depth / 1000.\n",
    "lib/datasets/tless/handle_test_data.py":
        "import tqdm\nimport os\nimport glob\nimport yaml\nfrom PIL import Image\nimport json\nimport numpy as np\n"
        "from lib.datasets.tless import opengl_renderer\nfrom lib.utils import base_utils\nimport cv2\n"
        "from lib.utils.tless import tless_config\n",
    "lib/datasets/tless/handle_ag_data.py":
        "import os\nimport json\nimport tqdm\nimport yaml\nfrom lib.utils import base_utils\nimport numpy as np\n"
        "from lib.datasets.tless import opengl_renderer\nfrom PIL import Image\nimport glob\nimport cv2\n",
    "lib/utils/__init__.py": "",
    "lib/utils/base_utils.py": "MARK = 'real base_utils'\n",
    "lib/utils/tless/__init__.py": "",
    "lib/utils/tless/tless_config.py": "visib_gt_min = 0.1\n",
}


def write_tless_checkout(tmp_path):
    for rel, text in TLESS_FILES.items():
        q = tmp_path / rel
        q.parent.mkdir(parents=True, exist_ok=True)
        q.write_text(text)
    return str(tmp_path)


def test_dropin_lets_the_tless_data_preparation_import_headless(tmp_path):
    """After install_tless_renderer_as_reference(), opengl_renderer, handle_test_data and handle_ag_data import without
    glumpy and bind this package's renderer; `lib.datasets` stays the real package and the depth drop-in is untouched."""
    tree = write_tless_checkout(tmp_path)
    code = f"""
        import sys
        sys.path.insert(0, {tree!r})
        import clean_pvnet_b200 as pvb
        pvb.install_tless_renderer_as_reference()
        from lib.datasets.tless import opengl_renderer, handle_test_data, handle_ag_data
        import lib.datasets
        assert lib.datasets.MARK == 'real datasets' and lib.datasets.__file__.startswith({tree!r})
        assert opengl_renderer.opengl_backend is pvb.render and handle_test_data.opengl_renderer is opengl_renderer
        assert handle_ag_data.opengl_renderer is opengl_renderer and handle_test_data.base_utils.MARK == 'real base_utils'
        assert 'lib.utils.renderer.opengl_utils' not in sys.modules
        pvb.install_tless_renderer_as_reference()
        print('ok')
    """
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=tree, env=dict(os.environ, PYTHONPATH=ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout
