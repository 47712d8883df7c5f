"""CPU tests of the DCNv2 twin (clean_pvnet_b200/dcn.py, csrc/dcn.cu): the fp64 restatement (oracle/dcn_oracle.py)
against torchvision's deform_conv2d and finite differences, the C ABI's validation, and the drop-in building the
unmodified DLA-34 CenterNet of a clean-pvnet checkout on this package without its THC extension."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import dcn_cases as dc
import dcn_oracle as do

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE = os.environ.get("PVNET_REFERENCE", "/root/reference")
DLA_DCN = os.path.join(REFERENCE, "lib", "networks", "ct", "dla_dcn.py")
tv_ops = pytest.importorskip("torchvision.ops")


def _tv(x, off, m, w, b, case):
    return tv_ops.deform_conv2d(x, off, w, b, stride=case.stride, padding=case.pad, dilation=case.dil, mask=m)


@pytest.mark.parametrize("case", dc.SWEEP, ids=dc.case_id)
def test_restatement_matches_torchvision_forward_and_autograd(case):
    """torchvision's deform_conv2d shares DCNv2's offset / mask layout and bilinear domain: in fp64 at non-integer
    sample points the restatement's forward and all five gradients agree with it to rounding."""
    x, off, m, w, b = dc.make_inputs(case, seed=7, offsets="random")
    out, _ = do.forward(x, off, m, w, b, case.stride, case.pad, case.dil, case.dg)
    t = [torch.from_numpy(a.astype(np.float64)).requires_grad_() for a in (x, off, m, w, b)]
    ref = _tv(*t, case)
    np.testing.assert_allclose(out, ref.detach().numpy(), rtol=1e-10, atol=1e-10)
    go = np.random.default_rng(3).standard_normal(ref.shape)
    ref.backward(torch.from_numpy(go))
    g = do.backward(x, off, m, w, b, go, case.stride, case.pad, case.dil, case.dg)
    for name, tt in zip(("grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"), t):
        np.testing.assert_allclose(g[name], tt.grad.numpy(), rtol=1e-9, atol=1e-9, err_msg=name)


@pytest.mark.parametrize("case", dc.SWEEP[:6], ids=dc.case_id)
def test_restatement_gradients_match_finite_differences(case):
    """Central differences of sum(grad_out * forward) away from kinks (sample points at least 1e-3 from a cell
    boundary): every gradient of the restatement is the derivative of its forward."""
    x, off, m, w, b = dc.make_inputs(case, seed=11, offsets="random")
    rng = np.random.default_rng(5)
    out, _ = do.forward(x, off, m, w, b, case.stride, case.pad, case.dil, case.dg)
    go = rng.standard_normal(out.shape)
    g = do.backward(x, off, m, w, b, go, case.stride, case.pad, case.dil, case.dg)
    args = [x, off, m, w, b]
    names = ["grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"]
    eps = 1e-6
    for k, name in enumerate(names):
        a = args[k].astype(np.float64)
        for idx in [tuple(rng.integers(0, s) for s in a.shape) for _ in range(6)]:
            def f(delta):
                aa = [v.astype(np.float64) for v in args]
                aa[k] = a.copy()
                aa[k][idx] += delta
                if k == 1:      # the restatement rounds sample points to fp32; stay in fp64 for the difference
                    return None
                return float((do.forward(*aa, case.stride, case.pad, case.dil, case.dg)[0] * go).sum())
            if k == 1:
                continue
            fd = (f(eps) - f(-eps)) / (2 * eps)
            assert abs(fd - g[name][idx]) <= 1e-5 * (1 + abs(fd)), (name, idx, fd, g[name][idx])


def test_offset_gradient_matches_finite_differences_in_fp64():
    """The offset gradient against central differences of torchvision's fp64 forward (the restatement itself rounds
    the sample point to fp32, as the reference does, so it cannot be differenced at 1e-6)."""
    case = dc.SWEEP[1]
    x, off, m, w, b = dc.make_inputs(case, seed=13, offsets="random")
    out, _ = do.forward(x, off, m, w, b, case.stride, case.pad, case.dil, case.dg)
    go = np.random.default_rng(2).standard_normal(out.shape)
    g = do.backward(x, off, m, w, b, go, case.stride, case.pad, case.dil, case.dg)["grad_offset"]
    t = [torch.from_numpy(a.astype(np.float64)) for a in (x, off, m, w, b)]
    rng = np.random.default_rng(1)
    for _ in range(8):
        idx = tuple(int(rng.integers(0, s)) for s in off.shape)
        vals = []
        for d in (1e-6, -1e-6):
            o = t[1].clone()
            o[idx] += d
            vals.append(float((_tv(t[0], o, t[2], t[3], t[4], case).numpy() * go).sum()))
        fd = (vals[0] - vals[1]) / 2e-6
        assert abs(fd - g[idx]) <= 1e-5 * (1 + abs(fd)), (idx, fd, g[idx])


def _desc(pvb, **kw):
    d = pvb._lib.PvbDcnDesc()
    base = dict(B=2, C=8, H=9, W=7, C_out=4, kh=3, kw=3, stride_h=1, stride_w=1, pad_h=1, pad_w=1, dilation_h=1,
                dilation_w=1, deformable_groups=1)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


BAD = [dict(B=-1), dict(C=0), dict(H=0), dict(W=-3), dict(C_out=0), dict(kh=0), dict(kw=-1), dict(stride_h=0),
       dict(stride_w=-1), dict(pad_h=-1), dict(pad_w=-2), dict(dilation_h=0), dict(dilation_w=-1),
       dict(deformable_groups=0), dict(deformable_groups=3), dict(C=6, deformable_groups=4),
       dict(kh=5, pad_h=0, H=4), dict(kw=3, dilation_w=4, pad_w=0, W=8), dict(B=65536),
       dict(H=65536, W=32768), dict(C=500000, kh=3, kw=3), dict(C_out=4194241),
       dict(kh=200, kw=200, H=300, W=300, pad_h=0, pad_w=0, C=2, deformable_groups=2),
       dict(H=2 ** 30, W=1), dict(dilation_h=2 ** 29, kh=3)]


@pytest.mark.parametrize("bad", BAD, ids=lambda b: ",".join(f"{k}={v}" for k, v in b.items()))
def test_bad_descriptors_are_rejected_before_any_cuda_call(pvb, bad):
    """Every malformed descriptor returns PVB_ERR_INVALID with a message and a zero workspace size; the pointers
    given are host garbage, so any CUDA call on them would fail differently."""
    lib = pvb._lib.load()
    d = _desc(pvb, **bad)
    junk = ctypes.c_void_p(16)
    assert lib.pvb_dcn_forward(ctypes.byref(d), *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID
    assert lib.pvb_last_error()
    assert lib.pvb_dcn_backward(ctypes.byref(d), *([junk] * 10), 1, junk, 1 << 40, None) == pvb._lib.PVB_ERR_INVALID
    assert lib.pvb_dcn_backward_workspace_bytes(ctypes.byref(d), 1) == 0
    assert lib.pvb_dcn_forward(None, *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID


def test_null_tensors_and_short_workspace_are_rejected(pvb):
    lib = pvb._lib.load()
    d = _desc(pvb)
    junk = ctypes.c_void_p(256)
    for k in range(6):
        ptrs = [junk] * 6
        ptrs[k] = None
        assert lib.pvb_dcn_forward(ctypes.byref(d), *ptrs, None) == pvb._lib.PVB_ERR_INVALID
    for k in range(10):
        ptrs = [junk] * 10
        ptrs[k] = None
        assert lib.pvb_dcn_backward(ctypes.byref(d), *ptrs, 1, junk, 1 << 40, None) == pvb._lib.PVB_ERR_INVALID
    need = lib.pvb_dcn_backward_workspace_bytes(ctypes.byref(d), 1)
    assert need >= 8 * 9 * 9 * 7 * 4          # one image's grad_cols
    assert lib.pvb_dcn_backward(ctypes.byref(d), *([junk] * 10), 1, junk, need - 1, None) == pvb._lib.PVB_ERR_WORKSPACE
    assert lib.pvb_dcn_backward(ctypes.byref(d), *([junk] * 10), 1, None, need, None) == pvb._lib.PVB_ERR_WORKSPACE
    assert lib.pvb_dcn_backward(ctypes.byref(d), *([junk] * 10), 1, ctypes.c_void_p(260), need, None) \
        == pvb._lib.PVB_ERR_WORKSPACE
    # B = 0 is a no-op: no tensor is read, none needs to exist
    d0 = _desc(pvb, B=0)
    assert lib.pvb_dcn_forward(ctypes.byref(d0), *([None] * 6), None) == 0
    assert lib.pvb_dcn_backward(ctypes.byref(d0), *([None] * 10), 1, None, 0, None) == 0
    # the chunk only changes grad_cols' share of the workspace
    assert lib.pvb_dcn_backward_workspace_bytes(ctypes.byref(d), 2) > need


def test_python_layer_rejects_cpu_and_non_fp32_inputs(pvb):
    case = dc.SWEEP[0]
    x, off, m, w, b = (torch.from_numpy(a) for a in dc.make_inputs(case, seed=1))
    with pytest.raises(RuntimeError, match="CUDA"):
        pvb.dcn_v2_conv(x, off, m, w, b, case.stride, case.pad, case.dil, case.dg)
    if torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="float32"):
            pvb.dcn_v2_conv(*(t.cuda().double() for t in (x, off, m, w, b)), case.stride, case.pad, case.dil, case.dg)


def test_module_surface_matches_the_reference(pvb):
    """Constructor signatures, parameter names and initialisation of DCNv2 / DCN (lib/networks/dcn_v2.py:57-128)."""
    import inspect
    for cls in (pvb.DCNv2, pvb.DCN):
        assert list(inspect.signature(cls.__init__).parameters) == [
            "self", "in_channels", "out_channels", "kernel_size", "stride", "padding", "dilation", "deformable_groups"]
    net = pvb.DCN(16, 8, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=2)
    assert sorted(net.state_dict()) == ["bias", "conv_offset_mask.bias", "conv_offset_mask.weight", "weight"]
    assert net.conv_offset_mask.out_channels == 2 * 3 * 9
    assert float(net.conv_offset_mask.weight.abs().sum()) == 0 and float(net.bias.abs().sum()) == 0
    assert float(net.weight.abs().max()) <= 1 / np.sqrt(16 * 9)
    assert not hasattr(pvb.dcn, "DCNPooling") and not hasattr(pvb.dcn, "DCNv2Pooling")


PROBE = r"""
import json, os, sys, types
ref = sys.argv[1]

def _no_network(*a, **k):
    raise RuntimeError("network access attempted")
import torch, torch.utils.model_zoo, torch.hub
torch.utils.model_zoo.load_url = _no_network
torch.hub.load_state_dict_from_url = _no_network

# stand-ins for `lib` and `lib.networks` whose __path__ points into the checkout: the real lib/networks/__init__.py
# imports make_network.py, which imports `imp` (gone in Python 3.12)
for name, path in (("lib", "lib"), ("lib.networks", "lib/networks")):
    mod = types.ModuleType(name)
    mod.__path__ = [os.path.join(ref, path)]
    sys.modules[name] = mod
sys.modules["lib"].networks = sys.modules["lib.networks"]

import clean_pvnet_b200 as pvb
pvb.install_dcn_as_reference_module()
import importlib.util
spec = importlib.util.spec_from_file_location("lib.networks.ct.dla_dcn", os.path.join(ref, "lib/networks/ct/dla_dcn.py"))
dla_dcn = importlib.util.module_from_spec(spec)
sys.modules[spec.name] = dla_dcn
spec.loader.exec_module(dla_dcn)
assert dla_dcn.DCN is pvb.DCN, dla_dcn.DCN

net = dla_dcn.DLASeg("dla34", {"ct_hm": 30, "wh": 2}, pretrained=False, down_ratio=4, final_kernel=1, last_level=5,
                     head_conv=256)
dcns = [m for m in net.modules() if type(m).__name__ in ("DCN", "DCNv2")]
assert all(type(m) is pvb.DCN for m in dcns)

recorded = []
def shape_only(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups):
    recorded.append([int(s) for s in input.shape[1:]] + [int(weight.shape[0])])
    B, _, H, W = input.shape
    return torch.empty((B, weight.shape[0], H, W), device=input.device)
pvb.dcn.dcn_v2_conv = shape_only
net = net.to("meta").eval()
out = {}
for (h, w) in [(544, 736), (480, 640), (512, 512)]:
    recorded.clear()
    net(torch.empty((1, 3, h, w), device="meta"))
    out[f"{h}x{w}"] = list(recorded)
print(json.dumps({"n": len(dcns), "ext": "lib.csrc.dcn_v2._ext" in sys.modules,
                  "dcn_keys": sorted(set(k.split(".conv.")[1] for k in net.state_dict() if k.startswith("dla_up") and ".conv." in k)),
                  "shapes": out}))
"""


@pytest.mark.skipif(not os.path.exists(DLA_DCN), reason="no clean-pvnet checkout")
def test_unmodified_dla_dcn_builds_on_this_package(tmp_path):
    """The checkout's own lib/networks/ct/dla_dcn.py, imported after install_dcn_as_reference_module(), builds the
    16-DCN DLA-34 CenterNet on pvb.DCN without importing lib.csrc.dcn_v2._ext or touching the network; the state_dict
    keys of each DCN are the reference's, and the (C, H, W, C_out) of every DCN call at 736x544, 640x480 and 512x512
    are dcn_cases.DETECTOR's, which pins the GPU tests to the detector's real shapes."""
    import json
    r = subprocess.run([sys.executable, "-c", PROBE, REFERENCE], cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["n"] == 16 and not res["ext"]
    assert res["dcn_keys"] == ["bias", "conv_offset_mask.bias", "conv_offset_mask.weight", "weight"]
    for key, shapes in res["shapes"].items():
        assert [tuple(s) for s in shapes] == dc.detector_shapes(key), (key, shapes)
