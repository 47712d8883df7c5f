"""CPU tests of the CenterNet decode (DESIGN.md 8j): the torch restatement against the reference's own decode
(tests/golden/ct_decode.npz, and live when PVNET_REFERENCE is set), the box un-crop restatement against the fixture,
argument validation of the C ABI and of the Python surface before any launch, workspace sizing, and the drop-in on a
miniature checkout next to the crop and DCN drop-ins."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import crop_cases as cc
import ct_decode_cases as dc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ct_decode.npz")


def test_restatement_equals_fixture():
    g = np.load(GOLDEN)
    assert list(g["names"]) == [c[0] for c in dc.golden_cases()]
    for c, (name, lg, wh, K) in enumerate(dc.golden_cases()):
        assert np.array_equal(lg, g[f"logits{c}"]) and np.array_equal(wh, g[f"wh{c}"]) and K == int(g[f"K{c}"]), name
        ct, det = dc.restate_decode(torch.from_numpy(lg), torch.from_numpy(wh), K)
        assert torch.equal(ct, torch.from_numpy(g[f"ct{c}"])), name
        assert torch.equal(det, torch.from_numpy(g[f"detection{c}"])), name


def test_fixture_is_tie_free_and_reaches_the_corners():
    g = np.load(GOLDEN)
    for c, name in enumerate(g["names"]):
        det = g[f"detection{c}"]
        for img in det:
            assert (np.diff(img[:, 4]) < 0).all(), name             # strictly decreasing scores: no ties anywhere
        lg = g[f"logits{c}"]
        H, W = lg.shape[2:]
        unclipped = dc.restate_decode(torch.from_numpy(lg), torch.from_numpy(g[f"wh{c}"]), int(g[f"K{c}"]), False)[1]
        assert (unclipped[..., 0] < 0).any() and (unclipped[..., 2] > W - 1).any(), name    # the clip bites
        assert (unclipped[..., 1] < 0).any() and (unclipped[..., 3] > H - 1).any(), name


def test_box_restatement_equals_fixture():
    g = np.load(GOLDEN)
    w, h = dc.BOX_INPUT_SIZE
    Minv = cc.crop_matrices(np.array(dc.BOX_CENTER, np.float32), np.float32(dc.BOX_SCALE[0]), w, h)[1]
    for c, name in enumerate(g["names"]):
        box = g[f"detection{c}"][..., :4] * np.float32(4)
        want = np.stack([np.stack([cc.dot_affine(b.reshape(-1, 2), Minv).ravel() for b in img]) for img in box])
        assert np.abs(want - g[f"boxes{c}"]).max() <= 1e-12, name


def test_restatement_equals_live_reference():
    ref = os.environ.get("PVNET_REFERENCE")
    if not ref:
        pytest.skip("PVNET_REFERENCE is not set")
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_golden_ct_decode as mg
    finally:
        sys.path.pop(0)
    du, cd = mg.reference_modules(ref)
    for name, lg, wh, K in dc.golden_cases(seed=7):
        hm = torch.from_numpy(lg)
        ct, det = cd.decode_ct_hm(torch.sigmoid(hm), torch.from_numpy(wh), K=K)
        det[..., :4] = du.clip_to_image(det[..., :4], hm.shape[2], hm.shape[3])
        mine = dc.restate_decode(hm, torch.from_numpy(wh), K)
        assert torch.equal(mine[0], ct) and torch.equal(mine[1], det), name


def _strides(*s):
    return (ctypes.c_int64 * 4)(*s)


def test_workspace_sizing(pvb):
    ws = pvb._lib.load().pvb_ct_decode_workspace_bytes
    # 32x32 tiles: 136x184 has 5 x 6 = 30 tiles; each keeps min(K, 1024) int64 keys, then K selected keys per image
    assert ws(1, 1, 136, 184, 100) == (30 * 100 * 8 + 255) // 256 * 256 + (100 * 8 + 255) // 256 * 256
    assert ws(32, 30, 104, 128, 100) == (32 * 30 * 16 * 100 * 8 + 255) // 256 * 256 + (32 * 100 * 8 + 255) // 256 * 256
    assert ws(2, 3, 40, 50, 2000) == (2 * 3 * 4 * 1024 * 8) + (2 * 2000 * 8 + 255) // 256 * 256
    assert ws(0, 3, 40, 50, 100) == 0
    assert ws(-1, 3, 40, 50, 100) == 0 and ws(1, 3, 40, 50, -1) == 0


def test_abi_validation(pvb):
    lib = pvb._lib
    f = lib.load().pvb_ct_decode
    p = ctypes.c_void_p(256)                                 # never dereferenced: validation precedes any CUDA call
    s4 = _strides(1000, 100, 10, 1)

    def call(B=1, C=1, H=10, W=10, K=5, clip=1, hm=p, hs=s4, wh=p, whs=s4, ct=p, det=p, ws=p, nbytes=1 << 20):
        return f(hm, hs, wh, whs, B, C, H, W, K, clip, ct, det, ws, nbytes, None)

    inv = lib.PVB_ERR_INVALID
    assert call(K=101) == inv                                # K > H*W: torch.topk raises
    assert call(K=0) == inv
    assert call(H=4096, W=4096) == inv                       # H*W = 2^24
    assert call(C=2000, K=10000, H=100, W=100) == inv        # C*K >= 2^24... and fine otherwise
    assert call(C=200, H=4000, W=4000, K=10) == inv          # C*H*W >= 2^31
    assert call(B=-1) == inv and call(B=65536) == inv and call(C=0) == inv and call(C=65536) == inv
    assert call(H=0) == inv and call(W=-3) == inv
    assert call(clip=2) == inv
    assert call(hs=None) == inv and call(whs=None) == inv
    assert call(hs=_strides(1000, 100, -10, 1)) == inv and call(whs=_strides(1000, 100, 10, -1)) == inv
    for k in ("hm", "wh", "ct", "det"):
        assert call(**{k: None}) == inv, k
    assert b"NULL" in lib.load().pvb_last_error()
    assert call(ws=None) == lib.PVB_ERR_WORKSPACE
    assert call(nbytes=16) == lib.PVB_ERR_WORKSPACE
    assert call(ws=ctypes.c_void_p(264)) == lib.PVB_ERR_WORKSPACE       # misaligned
    assert call(B=0, hm=None, wh=None, ct=None, det=None, ws=None) == lib.PVB_OK


def test_python_surface_rejects_bad_inputs(pvb):
    lg, wh = torch.zeros(1, 2, 8, 8), torch.zeros(1, 2, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        pvb.decode_detections(lg, wh)
    with pytest.raises(RuntimeError, match="CUDA"):
        pvb.decode_detections(lg.numpy(), wh)
    with pytest.raises(RuntimeError, match="detection"):
        pvb.detection_boxes(torch.zeros(2, 5), np.zeros((2, 2)), np.ones(2), (736, 544))
    with pytest.raises(RuntimeError, match="center"):
        pvb.detection_boxes(torch.zeros(2, 5, 6), np.zeros((3, 2)), np.ones(2), (736, 544))
    with pytest.raises(RuntimeError, match="scale"):
        pvb.detection_boxes(torch.zeros(2, 5, 6), np.zeros((2, 2)), np.ones(3), (736, 544))
    with pytest.raises(RuntimeError, match="float32"):
        pvb.detection_boxes(torch.zeros(2, 5, 6), np.zeros((2, 2)), np.array([720.0, 0.1]), (736, 544))


def test_python_checks_precede_any_launch(pvb, monkeypatch):
    """With stand-in CUDA tensors (the checks read only attributes), every refusal is raised before the library."""
    called = []
    monkeypatch.setattr(pvb.ct_decode, "_call", lambda *a: called.append(a))

    class Fake:
        def __init__(self, shape, dtype=torch.float32, device="cuda:0"):
            self.shape, self.dtype, self.device, self.is_cuda = torch.Size(shape), dtype, torch.device(device), True

        def dim(self):
            return len(self.shape)

    monkeypatch.setattr(pvb.ct_decode.torch, "Tensor", Fake)
    bad = [((Fake((1, 2, 8, 8), torch.float16), Fake((1, 2, 8, 8))), {}, "float32"),
           ((Fake((2, 8, 8)), Fake((1, 2, 8, 8))), {}, r"\[B,C,H,W\]"),
           ((Fake((1, 2, 8, 8)), Fake((1, 3, 8, 8))), {}, "wh must be"),
           ((Fake((1, 2, 8, 8)), Fake((1, 2, 8, 8), device="cuda:1")), {}, "one device"),
           ((Fake((1, 2, 8, 8)), Fake((1, 2, 8, 8))), {"K": 65}, "K must be in"),
           ((Fake((1, 2, 8, 8)), Fake((1, 2, 8, 8))), {"K": 2.0}, "K must be an int"),
           ((Fake((1, 2, 4096, 4096)), Fake((1, 2, 4096, 4096))), {}, "2\\^24"),
           ((Fake((1, 2000, 100, 100)), Fake((1, 2, 100, 100))), {"K": 9000}, "C\\*K")]
    for args, kw, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            pvb.decode_detections(*args, **kw)
    assert called == []


MINI = {
    "lib/__init__.py": "",
    "lib/config/__init__.py": "cfg = 'real cfg'\n",
    "lib/utils/__init__.py": "",
    "lib/utils/data_utils.py": "MARK = 'real data_utils'\n",
    "lib/networks/__init__.py": "",
    "lib/networks/ct/__init__.py": "",
    "lib/networks/ct/dla_dcn.py": "from lib.networks.dcn_v2 import DCN\nclass DLASeg:\n    pass\n",
    "lib/networks/ct/dla.py": textwrap.dedent("""
        from .dla_dcn import DLASeg
        from lib.utils import data_utils
        class Network:
            def decode_detection(self, output, h, w):
                return 'real decode'
            def forward(self, x, batch=None):
                return 'real forward'
        def get_network(*a):
            return Network()
    """),
    "lib/networks/ct_pvnet/__init__.py": "",
    "lib/networks/ct_pvnet/res.py": textwrap.dedent("""
        from lib.networks.ct.dla import get_network as get_pose_net
        def _crop(img, box, trans_output_inv, output):
            return 'real _crop'
        def crop(img, detection, batch, output):
            return 'real crop'
    """),
}


@pytest.mark.parametrize("order", [("dcn", "decode", "crop"), ("dcn", "crop", "decode")])
def test_install_patches_only_decode_detection(tmp_path, order):
    """A miniature checkout: after install_ct_decode_as_reference() ct.dla's Network.decode_detection is the fused one,
    everything else in ct.dla and the rest of `lib` stays the real thing, a second install changes nothing, and it
    works after the DCN drop-in with the crop drop-in before or after it."""
    for rel, text in MINI.items():
        q = tmp_path / rel
        q.parent.mkdir(parents=True, exist_ok=True)
        q.write_text(text)
    steps = {"dcn": "pvb.install_dcn_as_reference_module()", "decode": "pvb.install_ct_decode_as_reference()",
             "crop": "pvb.install_crop_as_reference()"}
    code = "\n".join([
        "import sys",
        f"sys.path.insert(0, {str(tmp_path)!r})",
        "import clean_pvnet_b200 as pvb",
        *[steps[s] for s in order],
        "from lib.networks.ct import dla",
        "from lib.networks.ct_pvnet import res",
        "from lib.config import cfg",
        "from lib.utils import data_utils",
        "import lib, lib.networks.dcn_v2 as dcn_v2",
        "assert dla.Network.decode_detection is pvb.ct_decode._decode_detection",
        "assert dla.Network().forward(None) == 'real forward' and dla.data_utils is data_utils",
        "assert res.get_pose_net is dla.get_network and res.crop is pvb.crop.cascade_crop",
        "assert res._crop(None, None, None, None) == 'real _crop' and cfg == 'real cfg'",
        "assert data_utils.MARK == 'real data_utils' and dcn_v2.DCN is pvb.dcn.DCN",
        f"assert lib.__file__.startswith({str(tmp_path)!r})",
        "pvb.install_ct_decode_as_reference()",
        "pvb.install_crop_as_reference()",
        "assert dla.Network.decode_detection is pvb.ct_decode._decode_detection and res.crop is pvb.crop.cascade_crop",
        "try:",
        "    dla.Network().decode_detection({'ct_hm': __import__('torch').zeros(1, 1, 4, 4),"
        " 'wh': __import__('torch').zeros(1, 2, 4, 4)}, 4, 4)",
        "except RuntimeError as e:",
        "    assert 'CUDA' in str(e), e",
        "print('ok')",
    ])
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout
