"""CPU tests of DCNv2's TF32 path (pvb_dcn_forward_tf32 / pvb_dcn_backward_tf32, csrc/dcn.cu; DESIGN.md section 8p):
a numpy restatement of the operand rounding, cvt.rna.tf32.f32; the dispatch on torch's matmul flag under every way of
setting it; the C ABI's refusals before any CUDA call; and the new kernels' register and shared-memory budget."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tf32_rna(x):
    """cvt.rna.tf32.f32 on fp32 bit patterns: keep 10 mantissa bits, round to nearest with ties away from zero (add
    half of the dropped 13 bits' weight to the magnitude, then truncate).  A carry moves into the exponent, so the
    largest finite values round to +-inf; subnormals round like normals (nothing is flushed); +-0 and +-inf stay;
    NaN stays NaN."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32)
    r = ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    return np.where(np.isnan(x), x, np.where(np.isinf(x), x, r)).astype(np.float32)


def _bits(*u):
    return np.array(u, dtype=np.uint32).view(np.float32)


def test_tf32_rna_rounds_ties_away_from_zero_for_both_signs():
    one_ulp = 2.0 ** -10                                      # TF32's spacing in [1, 2)
    x = np.array([1 + one_ulp / 2, -(1 + one_ulp / 2), 1 + 3 * one_ulp / 2, 1 + one_ulp / 2 - 2 ** -23,
                  1 + one_ulp / 2 + 2 ** -23], np.float32)
    want = np.array([1 + one_ulp, -(1 + one_ulp), 1 + 2 * one_ulp, 1, 1 + one_ulp], np.float32)
    assert np.array_equal(tf32_rna(x), want)


def test_tf32_rna_carries_into_the_exponent_and_overflows_to_inf():
    assert tf32_rna(_bits(0x3FFFF000))[0] == 2.0                       # 2 - 2^-11: a tie, away, to 2
    assert tf32_rna(_bits(0xBFFFF000))[0] == -2.0
    assert tf32_rna(_bits(0x3FFFEFFF))[0] == np.float32(2 - 2.0 ** -10)   # just below the tie
    big = np.finfo(np.float32).max
    assert np.array_equal(tf32_rna(np.array([big, -big], np.float32)), np.array([np.inf, -np.inf], np.float32))
    assert tf32_rna(_bits(0x7F7FEFFF))[0] == _bits(0x7F7FE000)[0]      # the largest value that stays finite


def test_tf32_rna_on_subnormals_zeros_infinities_and_nan():
    sub = tf32_rna(_bits(0x00000001, 0x00000FFF, 0x00001000, 0x80001000, 0x00002FFF, 0x007FF000, 0x007FFFFF))
    assert np.array_equal(sub.view(np.uint32), np.array(
        [0, 0, 0x2000, 0x80002000, 0x2000, 0x00800000, 0x00800000], np.uint32))
    z = tf32_rna(np.array([0.0, -0.0, np.inf, -np.inf], np.float32))
    assert np.array_equal(z.view(np.uint32), np.array([0, 0x80000000, 0x7F800000, 0xFF800000], np.uint32))
    assert np.isnan(tf32_rna(np.array([np.nan], np.float32))).all()
    x = np.random.default_rng(0).standard_normal(10000).astype(np.float32)
    r = tf32_rna(x)
    assert not (r.view(np.uint32) & 0x1FFF).any()
    assert (np.abs(r.astype(np.float64) - x) <= 2.0 ** -11 * np.abs(x)).all()


# ---- torch's flag, and which entry runs -----------------------------------------------------------------------------

def _save_flags():
    return torch.backends.fp32_precision, torch.backends.cuda.matmul.fp32_precision


def _restore_flags(saved):
    """Undoes the legacy routes first (allow_tf32 and set_float32_matmul_precision keep a state of their own that a
    legacy read checks against the new flags), then sets the saved values of the new flags."""
    torch.set_float32_matmul_precision("highest")
    torch.backends.fp32_precision, torch.backends.cuda.matmul.fp32_precision = saved


@pytest.fixture
def flags():
    """Restores torch's global and matmul fp32 precision exactly, so that later legacy reads (allow_tf32) work."""
    saved = _save_flags()
    yield
    _restore_flags(saved)


def _legacy_on():
    torch.backends.cuda.matmul.allow_tf32 = True


def _high():
    torch.set_float32_matmul_precision("high")


def _medium():
    torch.set_float32_matmul_precision("medium")


def _matmul_new():
    torch.backends.cuda.matmul.fp32_precision = "tf32"


def _global_new():
    torch.backends.fp32_precision = "tf32"


def _default():
    pass


def _ieee():
    torch.backends.cuda.matmul.fp32_precision = "ieee"


def _highest():
    torch.set_float32_matmul_precision("highest")


ON = [_legacy_on, _high, _medium, _matmul_new, _global_new]
OFF = [_default, _ieee, _highest]


@pytest.mark.parametrize("setter", ON + OFF, ids=lambda f: f.__name__.strip("_"))
def test_the_flag_read_follows_every_route_and_never_raises(pvb, flags, setter):
    setter()
    assert pvb.dcn.tf32_enabled() is (setter in ON)


@pytest.mark.parametrize("setter", ON + OFF, ids=lambda f: f.__name__.strip("_"))
def test_restoring_the_flags_lets_legacy_reads_work_again(flags, setter):
    saved = _save_flags()
    setter()
    _restore_flags(saved)
    assert _save_flags() == saved
    assert torch.backends.cuda.matmul.allow_tf32 is (saved[1] == "tf32")
    assert torch.get_float32_matmul_precision() == "highest"


@pytest.fixture
def calls(pvb, monkeypatch):
    """Records the entry of every _call; _check is bypassed so that CPU tensors reach the dispatch."""
    seen = []
    monkeypatch.setattr(pvb.dcn, "_check", lambda *a: None)
    monkeypatch.setattr(pvb.dcn, "_call", lambda entry, dev, *args: seen.append((entry, args)))
    return seen


def _tensors(dtype, channels_last):
    g = torch.Generator().manual_seed(0)
    lay = (lambda t: t.contiguous(memory_format=torch.channels_last)) if channels_last else (lambda t: t)
    x = lay(torch.randn((2, 8, 5, 6), generator=g)).to(dtype)
    off = lay(torch.randn((2, 18, 5, 6), generator=g))
    m = lay(torch.rand((2, 9, 5, 6), generator=g))
    return x, off, m, torch.randn((4, 8, 3, 3), generator=g), torch.randn((4,), generator=g)


DTYPE_IDS = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


class _CudaLooking(torch.Tensor):
    """A CPU tensor that passes dcn_backward's grad_output check, so that the stubbed dispatch is reached."""

    @property
    def is_cuda(self):
        return True


@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
@pytest.mark.parametrize("dt", list(DTYPE_IDS))
@pytest.mark.parametrize("setter", ON + OFF, ids=lambda f: f.__name__.strip("_"))
def test_which_entries_run_forward_and_backward(pvb, flags, calls, setter, dt, layout):
    """fp32: the TF32 forward and backward with the flag on, the FFMA ones with it off, in either layout.  fp16 / bf16:
    the forward is the half entry of its layout whatever the flag; the backward (fp32, on the up-casts) follows it."""
    setter()
    on = setter in ON
    x, off, m, w, b = _tensors(DTYPE_IDS[dt], layout == "channels_last")
    ops = pvb.dcn._operands(x, off, m, w, b)
    pvb.dcn.dcn_forward(x, *ops, 1, 1, 1, 1)
    if dt == "f32":
        fwd = "pvb_dcn_forward_tf32" if on else "pvb_dcn_forward"
    else:
        fwd = "pvb_dcn_forward_half_nhwc" if layout == "channels_last" else "pvb_dcn_forward_half"
    assert calls[-1][0] == fwd
    if fwd == "pvb_dcn_forward_tf32":        # the weight reaches the kernel tap-major, as the half kernels read it
        assert torch.equal(calls[-1][1][4], w.permute(0, 2, 3, 1).contiguous())
    up = [t.float() for t in (x, *ops)]
    go = torch.randn((2, 4, 5, 6)).as_subclass(_CudaLooking)
    pvb.dcn.dcn_backward(*up, go, 1, 1, 1, 1)
    assert calls[-1][0] == ("pvb_dcn_backward_tf32" if on else "pvb_dcn_backward")


# ---- the C ABI --------------------------------------------------------------------------------------------------------

def _desc(pvb, **kw):
    d = pvb._lib.PvbDcnDesc()
    base = dict(B=2, C=8, H=9, W=7, C_out=4, kh=3, kw=3, stride_h=1, stride_w=1, pad_h=1, pad_w=1, dilation_h=1,
                dilation_w=1, deformable_groups=1)
    base.update(kw)
    for k, v in base.items():
        setattr(d, k, v)
    return d


BAD = [dict(B=-1), dict(C=0), dict(C_out=0), dict(kh=0), dict(stride_w=0), dict(pad_h=-1), dict(dilation_w=0),
       dict(deformable_groups=3), dict(kh=5, pad_h=0, H=4), dict(B=65536), dict(C_out=4194241), dict(H=2 ** 30, W=1)]


@pytest.mark.parametrize("bad", BAD, ids=lambda b: ",".join(f"{k}={v}" for k, v in b.items()))
def test_bad_descriptors_are_rejected_before_any_cuda_call(pvb, bad):
    lib = pvb._lib.load()
    junk = ctypes.c_void_p(256)
    d = ctypes.byref(_desc(pvb, **bad))
    assert lib.pvb_dcn_forward_tf32(d, *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID
    assert lib.pvb_dcn_backward_tf32(d, *([junk] * 10), 1, junk, 1 << 30, None) == pvb._lib.PVB_ERR_INVALID
    assert lib.pvb_dcn_forward_tf32(None, *([junk] * 6), None) == pvb._lib.PVB_ERR_INVALID
    assert lib.pvb_dcn_backward_tf32(None, *([junk] * 10), 1, junk, 1 << 30, None) == pvb._lib.PVB_ERR_INVALID


def test_null_tensors_are_rejected_and_an_empty_batch_is_a_no_op(pvb):
    lib = pvb._lib.load()
    d = ctypes.byref(_desc(pvb))
    junk = ctypes.c_void_p(256)
    for k in range(6):
        ptrs = [junk] * 6
        ptrs[k] = None
        assert lib.pvb_dcn_forward_tf32(d, *ptrs, None) == pvb._lib.PVB_ERR_INVALID
        assert b"NULL" in lib.pvb_last_error()
    for k in range(10):
        ptrs = [junk] * 10
        ptrs[k] = None
        assert lib.pvb_dcn_backward_tf32(d, *ptrs, 1, junk, 1 << 30, None) == pvb._lib.PVB_ERR_INVALID
        assert b"NULL" in lib.pvb_last_error()
    empty = ctypes.byref(_desc(pvb, B=0))
    assert lib.pvb_dcn_forward_tf32(empty, *([None] * 6), None) == pvb._lib.PVB_OK
    assert lib.pvb_dcn_backward_tf32(empty, *([None] * 10), 1, None, 0, None) == pvb._lib.PVB_OK


def test_short_or_misaligned_workspace_is_refused_before_any_cuda_call(pvb):
    """The TF32 backward needs pvb_dcn_backward_workspace_bytes, the FFMA backward's plan."""
    lib = pvb._lib.load()
    d = _desc(pvb)
    need = lib.pvb_dcn_backward_workspace_bytes(ctypes.byref(d), 1)
    assert need > 0
    junk = ctypes.c_void_p(256)
    args = [junk] * 10
    assert lib.pvb_dcn_backward_tf32(ctypes.byref(d), *args, 1, junk, need - 1, None) == pvb._lib.PVB_ERR_WORKSPACE
    assert lib.pvb_dcn_backward_tf32(ctypes.byref(d), *args, 1, None, need, None) == pvb._lib.PVB_ERR_WORKSPACE
    assert lib.pvb_dcn_backward_tf32(ctypes.byref(d), *args, 1, ctypes.c_void_p(256 + 4), need, None) == \
        pvb._lib.PVB_ERR_WORKSPACE


# ---- the kernels' budget --------------------------------------------------------------------------------------------

def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


# registers (at most), static shared memory (exactly); DESIGN.md section 8p
BUDGET = {"dcn_forward_tf32_kernel": (112, 34816), "dcn_grad_cols_tf32_kernel": (128, 26624),
          "dcn_grad_weight_tf32_kernel": (120, 30720)}


@pytest.mark.skipif(_nvcc() is None, reason="no nvcc")
def test_tf32_kernels_fit_two_ctas_per_sm_without_spilling(tmp_path):
    src = os.path.join(ROOT, "clean_pvnet_b200", "csrc", "dcn.cu")
    r = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-cubin", "-o", str(tmp_path / "d.cubin"), src], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = r.stderr.splitlines()
    found = {}
    for i, line in enumerate(lines):
        if "Compiling entry function" not in line:
            continue
        for name in BUDGET:
            if name in line:
                assert "0 bytes spill stores, 0 bytes spill loads" in lines[i + 2], lines[i:i + 4]
                used = lines[i + 3]
                found[name] = (int(used.split("Used ")[1].split(" registers")[0]),
                               int(used.split("barriers, ")[1].split(" bytes smem")[0]))
    assert set(found) == set(BUDGET), r.stderr
    for name, (regs, smem) in found.items():
        assert regs <= BUDGET[name][0] and smem == BUDGET[name][1], (name, regs, smem)
        assert 2 * smem <= 228 * 1024 - 2 * 1024                   # two CTAs' shared memory fit an H100 SM
