"""CPU tests of the half-precision DCNv2 forward (pvb_dcn_forward_half, csrc/dcn.cu; DESIGN.md section 8n): the C ABI's
refusals before any CUDA call, the Python layer's dtype dispatch and refusals, and the kernels' register budget."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

import dcn_cases as dc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _desc(pvb, **kw):
    d = pvb._lib.PvbDcnDesc()
    base = dict(B=2, C=8, H=9, W=7, C_out=4, kh=3, kw=3, stride_h=1, stride_w=1, pad_h=1, pad_w=1, dilation_h=1,
                dilation_w=1, deformable_groups=1)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


BAD = [dict(B=-1), dict(C=0), dict(C_out=0), dict(kh=0), dict(stride_w=0), dict(pad_h=-1), dict(dilation_w=0),
       dict(deformable_groups=3), dict(kh=5, pad_h=0, H=4), dict(B=65536), dict(C_out=4194241),
       dict(H=2 ** 30, W=1)]


@pytest.mark.parametrize("bad", BAD, ids=lambda b: ",".join(f"{k}={v}" for k, v in b.items()))
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_bad_descriptors_are_rejected_before_any_cuda_call(pvb, bad, dtype):
    """The descriptor checks are pvb_dcn_forward's; the pointers are host garbage, so a CUDA call would fail otherwise."""
    lib = pvb._lib.load()
    code = pvb._lib.PVB_DCN_F16 if dtype == "f16" else pvb._lib.PVB_DCN_BF16
    junk = ctypes.c_void_p(16)
    assert lib.pvb_dcn_forward_half(ctypes.byref(_desc(pvb, **bad)), code, *([junk] * 6), None) == \
        pvb._lib.PVB_ERR_INVALID
    assert lib.pvb_last_error()
    assert lib.pvb_dcn_forward_half(None, code, *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID


@pytest.mark.parametrize("code", [0, 3, -1, 7])
def test_unknown_dtype_is_rejected_before_any_cuda_call(pvb, code):
    lib = pvb._lib.load()
    junk = ctypes.c_void_p(256)
    assert lib.pvb_dcn_forward_half(ctypes.byref(_desc(pvb)), code, *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID
    assert b"dtype" in lib.pvb_last_error()
    # B = 0 does not make an unknown dtype valid
    assert lib.pvb_dcn_forward_half(ctypes.byref(_desc(pvb, B=0)), code, *([None] * 6), None) == \
        pvb._lib.PVB_ERR_INVALID


def test_null_tensors_are_rejected_and_an_empty_batch_is_a_no_op(pvb):
    lib = pvb._lib.load()
    d = _desc(pvb)
    junk = ctypes.c_void_p(256)
    for code in (pvb._lib.PVB_DCN_F16, pvb._lib.PVB_DCN_BF16):
        for k in range(6):
            ptrs = [junk] * 6
            ptrs[k] = None
            assert lib.pvb_dcn_forward_half(ctypes.byref(d), code, *ptrs, None) == pvb._lib.PVB_ERR_INVALID
            assert b"NULL" in lib.pvb_last_error()
        assert lib.pvb_dcn_forward_half(ctypes.byref(_desc(pvb, B=0)), code, *([None] * 6), None) == pvb._lib.PVB_OK


def _inputs(dtype=torch.float32):
    case = dc.SWEEP[0]
    return case, [torch.from_numpy(a).to(dtype) for a in dc.make_inputs(case, seed=1)]


def test_python_layer_refuses_cpu_fp64_and_mixed_fp32_inputs(pvb):
    """CPU tensors, fp64, and an fp32 input with any half-precision operand are refused before a kernel is reached;
    the fp64 message still names float32."""
    case, (x, off, m, w, b) = _inputs()
    st = (case.stride, case.pad, case.dil, case.dg)
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        with pytest.raises(RuntimeError, match="CUDA"):
            pvb.dcn_v2_conv(x.to(dt), off, m, w, b, *st)
    with pytest.raises(RuntimeError, match="float32"):
        pvb.dcn_v2_conv(x.double(), off.double(), m.double(), w.double(), b.double(), *st)
    for k in range(1, 5):
        for dt in (torch.float16, torch.bfloat16):
            args = [x, off, m, w, b]
            args[k] = args[k].to(dt)
            with pytest.raises(RuntimeError, match="float32"):
                pvb.dcn_v2_conv(*args, *st)
    with pytest.raises(RuntimeError, match="float64"):          # a half input does not take fp64 operands
        pvb.dcn_v2_conv(x.bfloat16(), off, m, w.double(), b, *st)


def test_half_input_casts_the_other_operands_to_its_dtype(pvb):
    """offset, mask, weight and bias are rounded to nearest into the input's dtype, from fp32 or the other half type."""
    _, (x, off, m, w, b) = _inputs()
    for dt, other in ((torch.float16, torch.bfloat16), (torch.bfloat16, torch.float16)):
        ops = pvb.dcn._operands(x.to(dt), off, m.to(other), w, b)
        assert all(t.dtype == dt for t in ops)
        assert torch.equal(ops[0], off.to(dt)) and torch.equal(ops[2], w.to(dt))
        assert torch.equal(ops[1], m.to(other).to(dt))
    assert pvb.dcn._operands(x, off, m, w, b)[2] is w       # fp32: untouched


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


@pytest.mark.skipif(_nvcc() is None, reason="no nvcc")
def test_half_forward_kernels_do_not_spill(tmp_path):
    """Both instantiations fit two 256-thread CTAs per SM (<= 128 registers) without spilling."""
    src = os.path.join(ROOT, "clean_pvnet_b200", "csrc", "dcn.cu")
    r = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-cubin", "-o", str(tmp_path / "d.cubin"), src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    kernels = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "forward_half" in line]
    assert len(kernels) == 2, r.stderr
    for i in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 2], lines[i:i + 4]
        regs = int(lines[i + 3].split("Used ")[1].split(" registers")[0])
        assert regs <= 128, lines[i + 3]
