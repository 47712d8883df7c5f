"""CPU tests of the channels_last half-precision DCNv2 forward (pvb_dcn_forward_half_nhwc, csrc/dcn.cu; DESIGN.md
section 8o): the C ABI's refusals before any CUDA call, the Python layer's choice of entry point by the input's dtype and
layout, and the new kernels' register budget."""
import ctypes
import os
import subprocess

import pytest
import torch

from test_dcn_half_host import BAD, ROOT, _desc, _nvcc

CL = torch.channels_last


@pytest.mark.parametrize("bad", BAD, ids=lambda b: ",".join(f"{k}={v}" for k, v in b.items()))
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_bad_descriptors_are_rejected_before_any_cuda_call(pvb, bad, dtype):
    """The descriptor checks are pvb_dcn_forward_half's; the pointers are host garbage, so a CUDA call would fail."""
    lib = pvb._lib.load()
    code = pvb._lib.PVB_DCN_F16 if dtype == "f16" else pvb._lib.PVB_DCN_BF16
    junk = ctypes.c_void_p(16)
    assert lib.pvb_dcn_forward_half_nhwc(ctypes.byref(_desc(pvb, **bad)), code, *([junk] * 6), None) == \
        pvb._lib.PVB_ERR_INVALID
    assert lib.pvb_last_error()
    assert lib.pvb_dcn_forward_half_nhwc(None, code, *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID


@pytest.mark.parametrize("code", [0, 3, -1, 7])
def test_unknown_dtype_is_rejected_before_any_cuda_call(pvb, code):
    lib = pvb._lib.load()
    junk = ctypes.c_void_p(256)
    assert lib.pvb_dcn_forward_half_nhwc(ctypes.byref(_desc(pvb)), code, *([junk] * 6), None) == \
        pvb._lib.PVB_ERR_INVALID
    assert b"dtype" in lib.pvb_last_error()
    assert lib.pvb_dcn_forward_half_nhwc(ctypes.byref(_desc(pvb, B=0)), code, *([None] * 6), None) == \
        pvb._lib.PVB_ERR_INVALID


def test_null_tensors_are_rejected_and_an_empty_batch_is_a_no_op(pvb):
    lib = pvb._lib.load()
    d = _desc(pvb)
    junk = ctypes.c_void_p(256)
    for code in (pvb._lib.PVB_DCN_F16, pvb._lib.PVB_DCN_BF16):
        for k in range(6):
            ptrs = [junk] * 6
            ptrs[k] = None
            assert lib.pvb_dcn_forward_half_nhwc(ctypes.byref(d), code, *ptrs, None) == pvb._lib.PVB_ERR_INVALID
            assert b"NULL" in lib.pvb_last_error()
        assert lib.pvb_dcn_forward_half_nhwc(ctypes.byref(_desc(pvb, B=0)), code, *([None] * 6), None) == \
            pvb._lib.PVB_OK


def _operands(B=2, C=8, H=9, W=7, Co=4, dtype=torch.float16, layout=torch.contiguous_format):
    """Inputs of a 3x3, pad 1 call (Ho, Wo = H, W), input / offset / mask in `layout`."""
    g = torch.Generator().manual_seed(0)

    def laid_out(t):     # allocated in the layout: .contiguous() of an empty tensor would keep its strides
        return torch.empty(t.shape, dtype=dtype, memory_format=layout).copy_(t)
    x = laid_out(torch.randn((B, C, H, W), generator=g))
    off = laid_out(torch.randn((B, 18, H, W), generator=g))
    m = laid_out(torch.rand((B, 9, H, W), generator=g))
    w = torch.randn((Co, C, 3, 3), generator=g)
    b = torch.randn((Co,), generator=g)
    return x, off, m, w, b


@pytest.fixture
def calls(pvb, monkeypatch):
    """Records (entry, args) of every _call; _check is bypassed so that CPU tensors reach the dispatch."""
    seen = []
    monkeypatch.setattr(pvb.dcn, "_check", lambda *a: None)
    monkeypatch.setattr(pvb.dcn, "_call", lambda entry, dev, *args: seen.append((entry, args)))
    return seen


def _forward(pvb, x, off, m, w, b):
    return pvb.dcn.dcn_forward(x, off, m, w, b, 1, 1, 1, 1)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_a_channels_last_half_input_goes_to_the_nhwc_entry_without_a_copy(pvb, calls, dt):
    """The input itself reaches the kernel; offset and mask arrive channels_last from either layout (the same tensors
    when they are already channels_last); the output is channels_last."""
    for op_layout in (CL, torch.contiguous_format):
        x, off, m, w, b = _operands(dtype=dt, layout=CL)
        off, m = (t.contiguous(memory_format=op_layout) for t in (off, m))
        calls.clear()
        out = _forward(pvb, x, off, m, w, b)
        [(entry, args)] = calls
        assert entry == "pvb_dcn_forward_half_nhwc"
        assert args[1] == pvb.dcn.HALF[dt]
        xi, oi, mi, wi, bi, outi = args[2:]
        assert xi is x and outi is out
        assert out.is_contiguous(memory_format=CL) and not out.is_contiguous() and out.dtype == dt
        assert oi.is_contiguous(memory_format=CL) and mi.is_contiguous(memory_format=CL)
        assert torch.equal(oi, off) and torch.equal(mi, m)
        if op_layout is CL:
            assert oi.data_ptr() == off.data_ptr() and mi.data_ptr() == m.data_ptr()
        assert torch.equal(wi, w.to(dt).permute(0, 2, 3, 1).contiguous()) and torch.equal(bi, b.to(dt))


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_an_nchw_half_input_goes_to_the_nchw_entry(pvb, calls, dt):
    x, off, m, w, b = _operands(dtype=dt)
    out = _forward(pvb, x, off, m, w, b)
    assert [e for e, _ in calls] == ["pvb_dcn_forward_half"]
    assert out.is_contiguous()


@pytest.mark.parametrize("layout", [torch.contiguous_format, CL], ids=["nchw", "channels_last"])
def test_an_fp32_input_goes_to_the_fp32_entry_in_either_layout(pvb, calls, layout):
    x, off, m, w, b = _operands(dtype=torch.float32, layout=layout)
    out = _forward(pvb, x, off, m, w, b)
    [(entry, args)] = calls
    assert entry == "pvb_dcn_forward"
    assert all(t.is_contiguous() for t in args[1:]) and out.is_contiguous()


@pytest.mark.parametrize("shape", [dict(C=1), dict(H=1, W=1)], ids=["C1", "HW1"])
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_an_input_contiguous_in_both_layouts_goes_to_the_nchw_entry(pvb, calls, shape, dt):
    x, off, m, w, b = _operands(dtype=dt, layout=CL, **shape)
    assert x.is_contiguous() and x.is_contiguous(memory_format=CL)
    out = _forward(pvb, x, off, m, w, b)
    assert [e for e, _ in calls] == ["pvb_dcn_forward_half"]
    assert out.is_contiguous()


def test_an_empty_batch_calls_nothing_and_keeps_the_input_layout(pvb, calls):
    for layout, want_cl in ((CL, True), (torch.contiguous_format, False)):
        x, off, m, w, b = _operands(B=0, dtype=torch.bfloat16, layout=layout)
        out = _forward(pvb, x, off, m, w, b)
        assert calls == [] and out.shape == (0, 4, 9, 7) and out.dtype == torch.bfloat16
        assert (out.stride() == (9 * 7 * 4, 1, 7 * 4, 4)) == want_cl


@pytest.mark.skipif(_nvcc() is None, reason="no nvcc")
def test_nhwc_forward_kernels_do_not_spill(tmp_path):
    """Both instantiations fit two 256-thread CTAs per SM: <= 128 registers, no spills, and no more static shared
    memory than the NCHW kernel's 34 816 bytes."""
    src = os.path.join(ROOT, "clean_pvnet_b200", "csrc", "dcn.cu")
    r = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-cubin", "-o", str(tmp_path / "d.cubin"), src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    kernels = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "forward_nhwc" in line]
    assert len(kernels) == 2, r.stderr
    for i in kernels:
        assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 2], lines[i:i + 4]
        regs = int(lines[i + 3].split("Used ")[1].split(" registers")[0])
        assert regs <= 128, lines[i + 3]
        smem = int(lines[i + 3].split("barriers, ")[1].split(" bytes smem")[0])
        assert smem <= 34816, lines[i + 3]
