"""CPU tests of the deformable PSROI pooling twin (clean_pvnet_b200/dcn_pool.py, csrc/dcn_pool.cu): the fp64
restatement (oracle/dcn_pool_oracle.py) against finite differences and an analytic case, the C ABI's and the Python
layer's validation, the module surface against the reference's lib/networks/dcn_v2.py, the drop-in on a miniature
checkout, and the reference-kernel recipe."""
import ctypes
import importlib.util
import inspect
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import dcn_pool_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = os.environ.get("PVNET_REFERENCE", "/root/reference")
REF_DCN_PY = os.path.join(REFERENCE, "lib", "networks", "dcn_v2.py")
REF_POOL_CU = os.path.join(REFERENCE, "lib", "csrc", "dcn_v2", "src", "cuda", "dcn_v2_psroi_pooling_cuda.cu")


def _case(seed, n=3, B=2, C=4, H=12, W=14, P=3, ps=3, spp=2, nc=2):
    """ROIs well inside the map and samples at least 1e-3 from any integer, so the forward is smooth around them."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, C, H, W))
    for _ in range(100):
        rois = np.stack([rng.integers(0, B, n), rng.integers(8, 14, n), rng.integers(8, 14, n),
                         rng.integers(30, 36, n), rng.integers(26, 32, n)], 1).astype(np.float32)
        trans = (rng.uniform(-0.3, 0.3, (n, 2 * nc, ps, ps))).astype(np.float32)
        pts = po.points(rois, trans, B, H, W, P, ps, spp, nc, False, 0.25, 0.1, exact=True)
        d = np.concatenate([np.abs(pts[k] - np.round(pts[k])).ravel() for k in ("w", "h")])
        if d.min() > 1e-3 and pts["valid"].all():
            return x, rois, trans, dict(B=B, H=H, W=W, P=P, part_size=ps, spp=spp, num_classes=nc)
    raise AssertionError("no smooth case found")


def _pts(rois, trans, g, exact=True, no_trans=False):
    return po.points(rois, trans, g["B"], g["H"], g["W"], g["P"], g["part_size"], g["spp"], g["num_classes"], no_trans,
                     0.25, 0.1, exact=exact)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_restatement_gradients_match_central_differences(seed):
    """grad_input and grad_trans are the derivatives of the restatement's forward (fp64 sample points) at points at
    least 1e-3 from a cell boundary."""
    x, rois, trans, g = _case(seed)
    rng = np.random.default_rng(seed + 10)
    out, _, _ = po.forward(x, _pts(rois, trans, g))
    go = rng.standard_normal(out.shape)
    r = po.backward(x, _pts(rois, trans, g), go, 0.1)
    eps = 1e-6
    for _ in range(8):
        idx = tuple(int(rng.integers(0, s)) for s in x.shape)
        xp, xm = x.copy(), x.copy()
        xp[idx] += eps
        xm[idx] -= eps
        fd = ((po.forward(xp, _pts(rois, trans, g))[0] - po.forward(xm, _pts(rois, trans, g))[0]) * go).sum() / (2 * eps)
        assert abs(fd - r["grad_input"][idx]) <= 1e-6 * (1 + abs(fd)), (idx, fd, r["grad_input"][idx])
    t64 = trans.astype(np.float64)
    for _ in range(8):
        idx = tuple(int(rng.integers(0, s)) for s in trans.shape)
        tp, tm = t64.copy(), t64.copy()
        tp[idx] += eps
        tm[idx] -= eps
        fd = ((po.forward(x, _pts(rois, tp, g))[0] - po.forward(x, _pts(rois, tm, g))[0]) * go).sum() / (2 * eps)
        assert abs(fd - r["grad_trans"][idx]) <= 1e-6 * (1 + abs(fd)), (idx, fd, r["grad_trans"][idx])


def _indicator_bilinear(t, a, b):
    """Bilinear interpolation at t of the indicator of the integer pixels a..b."""
    return np.where((t >= a) & (t <= b), 1.0, np.where((t > a - 1) & (t < a), t - (a - 1),
                                                        np.where((t > b) & (t < b + 1), b + 1 - t, 0.0)))


@pytest.mark.parametrize("no_trans", [True, False])
def test_restatement_reproduces_the_constant_region_case(no_trans):
    """lib/csrc/dcn_v2/test.py's check_pooling_zero_offset: two constant squares, zero offsets.  Every output equals
    the mean over its bin's samples of the separable bilinear weight of the square, times its level."""
    x = np.zeros((2, 16, 64, 64))
    x[0, :, 16:26, 16:26] = 1.0
    x[1, :, 10:20, 20:30] = 2.0
    rois = np.array([[0, 65, 65, 103, 103], [1, 81, 41, 119, 79]], np.float32)
    trans = np.zeros((2, 2, 7, 7), np.float32)
    pts = po.points(rois, trans, 2, 64, 64, 7, 7, 4, 1, no_trans, 0.25, 0.0)
    out, count, _ = po.forward(x, pts)
    assert (count == 16).all()
    for r, (lev, (ya, yb), (xa, xb)) in enumerate([(1.0, (16, 25), (16, 25)), (2.0, (10, 19), (20, 29))]):
        val = lev * _indicator_bilinear(pts["w"][r, 0], xa, xb) * _indicator_bilinear(pts["h"][r, 0], ya, yb)
        want = val.mean(axis=-1)
        np.testing.assert_allclose(out[r], np.broadcast_to(want, out[r].shape), rtol=0, atol=1e-12)
    # the first ROI spans map columns 15.75 .. 25.5: its bins are inside the square but for the outer half-pixel
    assert out[0, :, 1:-1, 1:-1].min() == 1.0 and out[0].min() < 1.0


def _desc(pvb, **kw):
    d = pvb._lib.PvbDcnPoolDesc()
    base = dict(B=2, C=8, H=9, W=7, n_roi=3, output_dim=8, pooled_size=3, part_size=3, sample_per_part=2, group_size=1,
                num_classes=2, no_trans=0, spatial_scale=0.25, trans_std=0.1)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


BAD = [
    (dict(group_size=2), "group_size"), (dict(group_size=0), "group_size"),
    (dict(output_dim=4), "output_dim"), (dict(C=6, output_dim=6, num_classes=4), "multiple"),
    (dict(num_classes=0), "classes"), (dict(num_classes=3), "multiple"),
    (dict(B=-1), "shape"), (dict(C=0, output_dim=0), "shape"), (dict(H=0), "shape"), (dict(W=-2), "shape"),
    (dict(n_roi=-1), "shape"), (dict(pooled_size=0), "shape"), (dict(part_size=0), "shape"),
    (dict(sample_per_part=0), "sample_per_part"), (dict(sample_per_part=33), "sample_per_part"),
    (dict(n_roi=1 << 20, C=256, output_dim=256, pooled_size=7), "2^31"),
    (dict(B=64, C=256, output_dim=256, H=512, W=512), "2^31"),
    (dict(n_roi=1 << 20, pooled_size=1, part_size=1000, C=2, output_dim=2, num_classes=1), "2^31"),
]


@pytest.mark.parametrize("bad,why", BAD, ids=lambda b: ",".join(f"{k}={v}" for k, v in b.items())
                         if isinstance(b, dict) else b)
def test_bad_descriptors_are_rejected_before_any_cuda_call(pvb, bad, why):
    """Every malformed descriptor returns PVB_ERR_INVALID with a message naming the reason; the pointers are host
    garbage, so any CUDA call on them would fail differently."""
    lib = pvb._lib.load()
    d = _desc(pvb, **bad)
    junk = ctypes.c_void_p(16)
    assert lib.pvb_dcn_pool_forward(ctypes.byref(d), *([junk] * 5), None) == pvb._lib.PVB_ERR_INVALID
    assert why in lib.pvb_last_error().decode()
    assert lib.pvb_dcn_pool_backward(ctypes.byref(d), *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID
    assert why in lib.pvb_last_error().decode()
    assert lib.pvb_dcn_pool_forward(None, *([junk] * 5), None) == pvb._lib.PVB_ERR_INVALID


def test_null_tensors_are_rejected_and_empty_calls_are_no_ops(pvb):
    lib = pvb._lib.load()
    d = _desc(pvb)
    junk = ctypes.c_void_p(256)
    for k in range(4):                              # input, rois, trans, out (count may be NULL)
        ptrs = [junk] * 5
        ptrs[k] = None
        assert lib.pvb_dcn_pool_forward(ctypes.byref(d), *ptrs, None) == pvb._lib.PVB_ERR_INVALID
        assert "NULL" in lib.pvb_last_error().decode()
    for k in range(6):
        ptrs = [junk] * 6
        ptrs[k] = None
        assert lib.pvb_dcn_pool_backward(ctypes.byref(d), *ptrs, None) == pvb._lib.PVB_ERR_INVALID
    # trans and grad_trans are not read with no_trans; no ROI reads nothing and writes nothing
    d0 = _desc(pvb, n_roi=0, B=0)
    assert lib.pvb_dcn_pool_forward(ctypes.byref(d0), *([None] * 5), None) == 0
    assert lib.pvb_dcn_pool_backward(ctypes.byref(d0), *([None] * 6), None) == 0


def test_python_layer_rejects_cpu_non_fp32_and_bad_offsets(pvb):
    x = torch.zeros(2, 8, 9, 7)
    rois = torch.tensor([[0, 1, 1, 20, 20]], dtype=torch.float32)
    off = torch.zeros(1, 2, 3, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        pvb.dcn_v2_pooling(x, rois, off, 0.25, 3, 8, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        pvb.DCNv2Pooling(0.25, 3, 8, True)(x, rois, off)
    for bad in (torch.zeros(2, 2, 3, 3), torch.zeros(1, 3, 3, 3), torch.zeros(1, 2, 4, 4), torch.zeros(1, 2, 3)):
        with pytest.raises(RuntimeError, match="offset must be"):
            pvb.dcn_v2_pooling(x, rois, bad, 0.25, 3, 8, False)
    if torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="float32"):
            pvb.dcn_v2_pooling(x.cuda().double(), rois.cuda(), off.cuda(), 0.25, 3, 8, False)


def _reference_module():
    """The checkout's lib/networks/dcn_v2.py with its `_ext` import stubbed (it is never called here)."""
    saved = {k: sys.modules.get(k) for k in ("lib", "lib.csrc", "lib.csrc.dcn_v2", "lib.csrc.dcn_v2._ext")}
    try:
        for name in saved:
            mod = types.ModuleType(name)
            mod.__path__ = []
            sys.modules[name] = mod
        sys.modules["lib.csrc.dcn_v2"]._ext = sys.modules["lib.csrc.dcn_v2._ext"]
        spec = importlib.util.spec_from_file_location("ref_dcn_v2", REF_DCN_PY)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


@pytest.mark.skipif(not os.path.exists(REF_DCN_PY), reason="no clean-pvnet checkout")
def test_signatures_and_state_dict_match_the_reference(pvb):
    ref = _reference_module()
    pairs = [(ref._DCNv2Pooling.forward, pvb.dcn_pool._DCNv2Pooling.forward),
             (ref.DCNv2Pooling.__init__, pvb.DCNv2Pooling.__init__), (ref.DCNv2Pooling.forward, pvb.DCNv2Pooling.forward),
             (ref.DCNPooling.__init__, pvb.DCNPooling.__init__), (ref.DCNPooling.forward, pvb.DCNPooling.forward)]
    for a, b in pairs:
        assert inspect.signature(a) == inspect.signature(b), (a, b)
    for args in [(1 / 16, 7, 256, False), (0.25, 3, 8, True), (0.25, 7, 32, False, 1, None, 4, 0.1, 64)]:
        torch.manual_seed(0)
        theirs = ref.DCNPooling(*args)
        torch.manual_seed(0)
        ours = pvb.DCNPooling(*args)
        assert {k: v.shape for k, v in theirs.state_dict().items()} == {k: v.shape for k, v in ours.state_dict().items()}
        for k, v in theirs.state_dict().items():
            assert torch.equal(v, ours.state_dict()[k]), k      # same initialisation, draw for draw
        assert ours.load_state_dict(theirs.state_dict()) is not None
        for name in ("spatial_scale", "pooled_size", "output_dim", "no_trans", "group_size", "part_size",
                     "sample_per_part", "trans_std", "deform_fc_dim"):
            assert getattr(ours, name) == getattr(theirs, name), name


MINI = {
    "lib/__init__.py": "",
    "lib/networks/__init__.py": "",
    "lib/networks/dcn_v2.py": "from lib.csrc.dcn_v2 import _ext as _backend\n",
    "lib/csrc/__init__.py": "",
    "lib/csrc/dcn_v2/__init__.py": "",
    "lib/csrc/dcn_v2/_ext.py": "raise ImportError('the THC extension is not built')\n",
}


def test_install_binds_all_six_names_on_a_miniature_checkout(tmp_path):
    for rel, text in MINI.items():
        q = tmp_path / rel
        q.parent.mkdir(parents=True, exist_ok=True)
        q.write_text(text)
    code = "\n".join([
        "import sys",
        f"sys.path.insert(0, {str(tmp_path)!r})",
        "import clean_pvnet_b200 as pvb",
        "m = pvb.install_dcn_as_reference_module()",
        "from lib.networks.dcn_v2 import dcn_v2_pooling, DCNv2Pooling, DCNPooling",
        "from lib.networks.dcn_v2 import dcn_v2_conv, DCNv2, DCN",
        "import lib, lib.networks",
        "assert DCNPooling is pvb.DCNPooling and DCN is pvb.DCN and dcn_v2_pooling is pvb.dcn_v2_pooling",
        "assert lib.networks.dcn_v2 is m and pvb.install_dcn_as_reference_module() is m",
        f"assert lib.__file__.startswith({str(tmp_path)!r})",
        "assert 'lib.csrc.dcn_v2._ext' not in sys.modules",
        "print('ok')",
    ])
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


@pytest.mark.skipif(not os.path.exists(REF_POOL_CU) or _nvcc() is None, reason="no clean-pvnet checkout or no nvcc")
def test_reference_recipes_build_both_libraries(tmp_path):
    """oracle/build_dcn_ref.py and oracle/build_dcn_pool_ref.py, pointed at a scratch output, build both reference
    libraries, and the pooling one exports its two launchers."""
    for script, lib in (("build_dcn_ref.py", "libdcn_ref.so"), ("build_dcn_pool_ref.py", "libdcn_pool_ref.so")):
        spec = importlib.util.spec_from_file_location("recipe_" + lib, os.path.join(ROOT, "oracle", script))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mod.OUT, mod.LIB = str(tmp_path), str(tmp_path / lib)
        assert mod.build(force=True)
        assert (tmp_path / lib).stat().st_size > 0
    syms = subprocess.run(["nm", "-D", str(tmp_path / "libdcn_pool_ref.so")], capture_output=True, text=True).stdout
    assert "ref_dcn_pool_forward" in syms and "ref_dcn_pool_backward" in syms


@pytest.mark.skipif(_nvcc() is None, reason="no nvcc")
def test_pool_kernels_do_not_spill(tmp_path):
    src = os.path.join(ROOT, "clean_pvnet_b200", "csrc", "dcn_pool.cu")
    r = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-cubin", "-o", str(tmp_path / "p.cubin"), src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    kernels = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "dcn_pool" in line]
    assert len(kernels) == 2, r.stderr
    for i in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 2], lines[i:i + 4]
