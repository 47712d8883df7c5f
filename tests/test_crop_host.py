"""CPU tests of T-LESS's PVNet crop (DESIGN.md 8g): the numpy restatement of the warp and of the crop matrix
(tests/crop_cases.py) against cv2 byte for byte and bit for bit, the restatement against the reference's own
pvnet_transform / un-crop outputs (tests/golden/tless_crop.npz), the C ABI's argument validation, and the cascade drop-in
on a miniature checkout."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import crop_cases as cc

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "tless_crop.npz")
SIZES = [(128, 128), (256, 256), (192, 144)]


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def test_warp_restatement_equals_cv2_byte_for_byte():
    print("cv2", cv2.__version__)
    rng = np.random.default_rng(7)
    imgs = cc.random_images(rng, 3)
    boxes = np.concatenate([cc.random_boxes(rng, 96), cc.DEGENERATE])
    for i, b in enumerate(boxes):
        w, h = SIZES[i % len(SIZES)]
        img = imgs[i % len(imgs)]
        c, s = cc.center_scale(b, 2.4 if i % 2 else 1.2)
        M, _ = cc.crop_matrices(c, s, w, h)
        want = cv2.warpAffine(img, M, (w, h), flags=cv2.INTER_LINEAR)
        assert np.array_equal(cc.warp_linear(img, M, w, h), want), (i, b)


def test_warp_restatement_full_image_resize_and_one_channel():
    """The detector's full-image resize (tless_test_utils.augment: 720x540 -> 736x544) and a single-channel image."""
    rng = np.random.default_rng(8)
    img = cc.random_images(rng, 1)[0]
    c = np.array([360.0, 270.0], np.float32)
    src, dst = cc.crop_points(c, 720.0, 736, 544)
    M = cv2.getAffineTransform(src, dst)
    assert np.array_equal(cc.warp_linear(img, M, 736, 544), cv2.warpAffine(img, M, (736, 544), flags=cv2.INTER_LINEAR))
    g = np.ascontiguousarray(img[:, :, 1])
    assert np.array_equal(cc.warp_linear(g, M, 97, 61), cv2.warpAffine(g, M, (97, 61), flags=cv2.INTER_LINEAR))


def test_lu_restatement_equals_get_affine_transform_bit_for_bit():
    rng = np.random.default_rng(9)
    n = 0
    for i in range(3000):
        b = rng.uniform(-100, 800, 4) if i % 3 else rng.integers(-100, 800, 4).astype(np.float64) + 0.5 * (i % 2)
        b = [min(b[0], b[2]), min(b[1], b[3]), max(b[0], b[2]), max(b[1], b[3])]
        w, h = SIZES[i % len(SIZES)]
        c, s = cc.center_scale(b, (2.4, 1.2, 1.8)[i % 3], center_f32=bool(i % 4))
        src, dst = cc.crop_points(c, s, w, h)
        for a, z in ((src, dst), (dst, src)):
            assert np.array_equal(_bits(cc.get_affine(a, z)), _bits(cv2.getAffineTransform(a, z))), (i, b)
            n += 1
    assert n == 6000


def test_degenerate_box_is_what_cv2_does():
    """A zero-size box makes the system singular: cv2 returns an all-zero forward matrix, the warp then samples pixel
    (0, 0) everywhere, and the magnified box shrinks to pixel (0, 0) of the crop."""
    img = cc.random_images(np.random.default_rng(10), 1)[0]
    for b in cc.DEGENERATE:
        c, s = cc.center_scale(b, 2.4)
        src, dst = cc.crop_points(c, s, 256, 256)
        M = cv2.getAffineTransform(src, dst)
        assert not M.any() and not cc.get_affine(src, dst).any()
        assert np.array_equal(_bits(cc.get_affine(dst, src)), _bits(cv2.getAffineTransform(dst, src)))
        inp, u8, *_ = cc.crop_restated(img, b)
        assert np.array_equal(u8[0, 0], img[0, 0]) and not u8.reshape(-1, 3)[1:].any()


def test_restatement_equals_the_reference_pvnet_transform():
    g = np.load(GOLDEN)
    img = cc.pattern_images(g["img_params"])
    for name in cc.CONFIGS:
        w, h, scale_ratio, box_ratio = g[f"{name}_config"]
        w, h = int(w), int(h)
        boxes, index = g[f"{name}_boxes"], g[f"{name}_index"]
        assert len(boxes) >= 12 and any(b[2] == b[0] for b in boxes)
        for i, (b, k) in enumerate(zip(boxes, index)):
            inp, u8, c, s, M, Minv = cc.crop_restated(img[k], b, (w, h), scale_ratio, box_ratio)
            assert np.array_equal(u8, g[f"{name}_crop"][i]), (name, i)
            assert cc.sha256(inp) == g[f"{name}_inp_sha256"][i], (name, i)
            assert np.array_equal(c.astype(np.float32), g[f"{name}_center"][i]) and s == g[f"{name}_scale"][i]
            un = cc.uncrop_restated(g[f"{name}_kpt"][i], g[f"{name}_center"][i], s, (w, h))
            assert np.abs(un - g[f"{name}_uncrop"][i]).max() <= 1e-12, (name, i)


# ---- C ABI, without a GPU ---------------------------------------------------------------------------------------------

def test_crop_abi_validation(pvb):
    lib = pvb._lib.load()
    INV, OK = pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_OK
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    st = (ctypes.c_int64 * 4)(540 * 720 * 3, 720 * 3, 3, 1)
    ms = (ctypes.c_float * 3)(*cc.MEAN)
    sd = (ctypes.c_float * 3)(*cc.STD)
    ok = [p, 1, 540, 720, st, p, None, 2, 256, 256, 2.4, 1.2, 1, ms, sd, p, None, p, p, p, None]
    ci = lambda a: lib.pvb_crop_inputs(*a, None)   # noqa: E731
    for i, bad in ((1, -1), (2, 0), (3, 40000), (7, -1), (8, 0), (10, float("nan")), (11, -1.0), (12, 8)):
        a = list(ok); a[i] = bad
        assert ci(a) == INV, i
    for i in (0, 4, 5, 13, 14, 15, 17, 18, 19):
        a = list(ok); a[i] = None
        assert ci(a) == INV, i
    a = list(ok); a[4] = (ctypes.c_int64 * 4)(-1, 0, 0, 0)
    assert ci(a) == INV
    sd0 = (ctypes.c_float * 3)(1.0, 0.0, 1.0)
    a = list(ok); a[14] = sd0
    assert ci(a) == INV
    a = list(ok); a[7] = 0
    assert ci(a) == OK                                                       # n == 0: no-op
    un = [p, p, p, 2, 9, 256, 256, p]
    assert lib.pvb_uncrop_keypoints(*un[:3], -1, *un[4:], None) == INV
    assert lib.pvb_uncrop_keypoints(*un[:5], 0, *un[6:], None) == INV
    assert lib.pvb_uncrop_keypoints(None, *un[1:], None) == INV
    assert lib.pvb_uncrop_keypoints(*un[:3], 0, *un[4:], None) == OK
    wa = [p, 1, 540, 720, 3, st, p, None, 2, 256, 256, p]
    assert lib.pvb_warp_affine_linear(*wa[:4], 5, *wa[5:], None) == INV      # 1..4 channels
    assert lib.pvb_warp_affine_linear(*wa[:6], None, *wa[7:], None) == INV
    assert lib.pvb_warp_affine_linear(*wa[:8], 0, *wa[9:], None) == OK
    assert len(lib.pvb_last_error()) > 0


def test_python_errors_before_any_launch(pvb):
    img = np.zeros((54, 72, 3), np.uint8)
    with pytest.raises(RuntimeError, match="img"):
        pvb.crop_inputs(np.zeros((54, 72), np.uint8), np.zeros((1, 4)))
    with pytest.raises(RuntimeError, match="boxes"):
        pvb.crop_inputs(img, np.zeros((1, 3)))
    with pytest.raises(RuntimeError, match="image_index"):
        pvb.crop_inputs(np.zeros((2, 54, 72, 3), np.uint8), np.zeros((1, 4)))
    with pytest.raises(RuntimeError, match="kpt_2d"):
        pvb.uncrop_keypoints(np.zeros((2, 9)), np.zeros((2, 2)), np.ones(2), (256, 256))
    with pytest.raises(RuntimeError, match="M"):
        pvb.warp_affine_batch(img, np.zeros((1, 3, 3)), (8, 8))
    assert pvb.crop.crop_inputs is pvb.crop_inputs


def test_install_crop_patches_only_crop(tmp_path):
    """A miniature checkout of lib/networks/ct_pvnet/res.py: after install_crop_as_reference() the module's `crop` is the
    device crop and everything else in it, and the rest of `lib`, stays the real thing."""
    files = {
        "lib/__init__.py": "",
        "lib/config/__init__.py": "cfg = 'real cfg'\n",
        "lib/utils/data_utils.py": "MARK = 'real data_utils'\n",
        "lib/networks/__init__.py": "",
        "lib/networks/ct_pvnet/__init__.py": "",
        "lib/networks/ct_pvnet/res.py": textwrap.dedent("""
            from lib.config import cfg
            from lib.utils import data_utils
            def _crop(img, box, trans_output_inv, output):
                return 'real _crop'
            def crop(img, detection, batch, output):
                return 'real crop'
            class Network:
                def forward(self, x, batch=None):
                    return crop(None, None, batch, {})
        """),
    }
    for rel, text in files.items():
        q = tmp_path / rel
        q.parent.mkdir(parents=True, exist_ok=True)
        q.write_text(text)
    code = f"""
        import sys
        sys.path.insert(0, {str(tmp_path)!r})
        import clean_pvnet_b200 as pvb
        pvb.install_crop_as_reference()
        from lib.networks.ct_pvnet import res
        from lib.config import cfg
        from lib.utils import data_utils
        assert res.crop is pvb.crop.cascade_crop, res.crop
        assert res._crop(None, None, None, None) == 'real _crop' and cfg == 'real cfg'
        assert data_utils.MARK == 'real data_utils' and res.data_utils is data_utils
        import lib
        assert lib.__file__.startswith({str(tmp_path)!r})
        pvb.install_crop_as_reference()
        assert res.crop is pvb.crop.cascade_crop
        print('ok')
    """
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout
