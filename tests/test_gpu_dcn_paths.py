"""GPU tests of DCNv2 (csrc/dcn.cu) at the small shapes of tests/dcn_paths.py, which between them take every side of the
half-precision forward's load-path and tile-tail branches: the 16-byte weight and NHWC corner loads, partial last K
chunks, several deformable groups, partly filled output tiles, every split-K factor from 1 to 8.  Each is checked
against a reference that shares no code with the path under test: the columns against the reference's im2col bit for
bit, the product against fp64 within DESIGN.md section 8n's bound, the fp32 kernels against the fp64 restatement.

Weights and inputs sit between NaN guard bands, so a read past a tensor's end (a zero-fill gone, a guard off by a
chunk) turns the output NaN instead of multiplying a neighbour's finite values by the zero columns of a padded chunk.
The half-precision weight is passed channels_last, which is the tap-major layout the kernel reads, so the kernel gets
the guarded storage itself rather than a copy."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import dcn_cases as dc
import dcn_oracle as do
import dcn_paths as dp
from test_gpu_dcn import U, _chains, gamma, gpu, ref_cols
from test_gpu_dcn_half import C_BOUND, DT_IDS, DTYPES, UNIT, fwd, lowp
from test_gpu_dcn_half import test_backward_is_the_fp32_backward_on_the_up_cast_operands as half_backward_check
from test_gpu_dcn_nhwc import assert_bitwise_channels_last

pytestmark = pytest.mark.gpu
CL = torch.channels_last
FORMATS = {"nchw": torch.contiguous_format, "channels_last": CL}
GUARD = 64        # NaN elements on each side of a guarded tensor: 128 bytes in fp16 / bf16, so the data stays aligned


def guarded(t, memory_format=torch.contiguous_format, shift=0):
    """t's values, laid out in memory_format, in a buffer that holds NaN in the GUARD elements before and after them;
    the data starts `shift` elements past a 16-byte boundary."""
    n = t.numel()
    buf = torch.full((2 * GUARD + shift + n,), float("nan"), dtype=t.dtype, device=t.device)
    g = buf[GUARD + shift:GUARD + shift + n].as_strided(t.shape, t.contiguous(memory_format=memory_format).stride())
    return g.copy_(t)


def tap_major(w):
    """A guarded half-precision weight that the forward passes to the kernel uncopied: channels_last [C_out, C, kh, kw]
    is the tap-major [C_out, kh, kw, C] the kernel reads."""
    g = guarded(w, CL)
    assert g.permute(0, 2, 3, 1).is_contiguous()
    return g


def run(pvb, c, x, off, m, w, b, layout, shift=0):
    """The forward on a guarded input (and offset, mask) in `layout`, with the weight tap_major."""
    f = FORMATS[layout]
    return fwd(pvb, c, guarded(x, f, shift), off.contiguous(memory_format=f), m.contiguous(memory_format=f),
               tap_major(w), b)


def product_bound(c, x, off, m, w, b, dt):
    """E = fp64(b + W col) on the rounded operands, and the bound of DESIGN.md section 8n on |out - E|."""
    cols = ref_cols(c, x.float(), off.float(), m.float()).to(dt)
    W2 = w.reshape(c.Co, -1)
    exact = b.double()[None, :, None] + torch.matmul(W2.double(), cols.double())
    absb = b.double().abs()[None, :, None] + torch.matmul(W2.double().abs(), cols.double().abs())
    return exact, C_BOUND * c.C * c.kh * c.kw * U * absb + UNIT[dt] * exact.abs()


def assert_within(out, c, exact, bound):
    err = (out.reshape(c.B, c.Co, -1).double() - exact).abs()
    assert bool((err <= bound).all()), float((err / bound.clamp_min(1e-300)).nan_to_num(float("inf")).max())


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("offsets", ["edges", "random"])
@pytest.mark.parametrize("case", dp.PATHS, ids=dc.case_id)
def test_identity_weight_returns_the_rounded_reference_columns_in_both_layouts(pvb, case, offsets, dt):
    """W = I (C_out = C*kh*kw, two or more output tiles), bias 0: the output is to(dtype) of the reference im2col on the
    up-cast inputs, exactly, in both layouts; "edges" puts sample points on every edge of the bilinear domain and at
    NaN / +-inf."""
    dt = DTYPES[dt]
    x, off, m, _, _ = dc.make_inputs(case, seed=21, offsets=offsets, nonfinite=True)
    wid, bid = dc.identity_weight(case)
    x, off, m, wid, bid = lowp((x, off, m, wid, bid), dt)
    ic = case._replace(Co=wid.shape[0])
    want = ref_cols(case, x.float(), off.float(), m.float()).to(dt)
    for layout in dp.LAYOUTS:
        ours = run(pvb, ic, x, off, m, wid, bid, layout)
        assert ours.dtype == dt and ours.is_contiguous(memory_format=FORMATS[layout])
        ours = ours.reshape(want.shape)
        assert torch.equal(ours, want), (layout, float((ours.float() - want.float()).abs().nan_to_num(1e30).max()))


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case", dp.PATHS, ids=dc.case_id)
def test_product_is_within_the_tensor_core_bound_and_the_same_in_both_layouts(pvb, case, dt):
    """Real weights: both layouts meet the bound against fp64 b + W cols on the rounded operands, and the
    channels_last output is the NCHW output bit for bit."""
    dt = DTYPES[dt]
    x, off, m, w, b = lowp(dc.make_inputs(case, seed=3, offsets="random"), dt)
    exact, bound = product_bound(case, x, off, m, w, b, dt)
    out = {layout: run(pvb, case, x, off, m, w, b, layout) for layout in dp.LAYOUTS}
    for o in out.values():
        assert_within(o, case, exact, bound)
    assert_bitwise_channels_last(out["channels_last"], out["nchw"])


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case", dp.PATHS, ids=dc.case_id)
def test_a_misaligned_channels_last_input_gives_the_aligned_bits(pvb, case, dt):
    """A channels_last input whose data starts 2 bytes past a 16-byte boundary still runs the NHWC kernel, on its
    scalar sampler, and returns the 16-byte sampler's output bit for bit, within the bound."""
    dt = DTYPES[dt]
    x, off, m, w, b = lowp(dc.make_inputs(case, seed=3, offsets="random"), dt)
    xm = guarded(x, CL, shift=1)
    assert xm.data_ptr() % 16 == 2 and pvb.dcn._nhwc(xm)
    want = run(pvb, case, x, off, m, w, b, "channels_last")
    got = run(pvb, case, x, off, m, w, b, "channels_last", shift=1)
    assert_bitwise_channels_last(got, want)
    assert_within(got, case, *product_bound(case, x, off, m, w, b, dt))


@pytest.mark.parametrize("offsets", ["edges", "random"])
@pytest.mark.parametrize("case", dp.PATHS, ids=dc.case_id)
def test_fp32_forward_is_within_the_rounding_bound_of_the_restatement(pvb, case, offsets):
    """|ours - fp64| <= gamma_{K+9} (|b| + sum |W| |col|): K + 1 roundings for the bias and the K products' sum, 8
    for a column entry sampled in fp32 (its bilinear weights, the four-term blend and the mask)."""
    arrs = dc.make_inputs(case, seed=3, offsets=offsets, nonfinite=True)
    want, want_abs = do.forward(*arrs, case.stride, case.pad, case.dil, case.dg)
    x, off, m, w, b = gpu(*arrs)
    ours = fwd(pvb, case, guarded(x), off, m, guarded(w), b).double().cpu().numpy()
    bound = gamma(case.C * case.kh * case.kw + 9) * want_abs
    err = np.abs(ours - want)
    assert (err <= bound).all(), float((err / np.maximum(bound, 1e-300)).max())


@pytest.mark.parametrize("B", dp.BACKWARD_BATCHES)
@pytest.mark.parametrize("case", dp.BACKWARD, ids=dc.case_id)
def test_fp32_backward_is_within_the_rounding_bound_in_one_chunk_and_in_pairs(pvb, case, B):
    """All five gradients against the fp64 restatement, with grad_cols in one chunk of B images and in chunks of 2
    (the last one image, at b0 = B - 1); only grad_input, summed with float atomics, may differ between the two."""
    case = case._replace(B=B)
    arrs = dc.make_inputs(case, seed=9, offsets="random")
    Ho, Wo = dc.out_hw(case)
    go = np.random.default_rng(4).standard_normal((B, case.Co, Ho, Wo)).astype(np.float32)
    want = do.backward(*arrs, go, case.stride, case.pad, case.dil, case.dg)
    t = gpu(*arrs, go)
    per_image = case.C * case.kh * case.kw * Ho * Wo * 4
    one = pvb.dcn.dcn_backward(*t, case.stride, case.pad, case.dil, case.dg, max_column_bytes=B * per_image)
    pairs = pvb.dcn.dcn_backward(*t, case.stride, case.pad, case.dil, case.dg, max_column_bytes=2 * per_image)
    names = ["grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias"]
    chains = _chains(case)
    for name, g1, g2 in zip(names, one, pairs):
        if name == "grad_input":
            n = case.Co + 8 + want["grad_input_terms"]
        else:
            n = chains[name]
            assert torch.equal(g1, g2), name
        bound = n * U * want[name + "_abs"] * 1.01 + 1e-30
        for g in (g1, g2):
            err = np.abs(g.double().cpu().numpy() - want[name])
            assert (err <= bound).all(), (name, float((err / bound).max()))


HALF_BWD = [dp.PATHS[3], dp.PATHS[4]]       # two groups of 8 channels, C_out 200; four groups of 16, C_out 257


@pytest.mark.parametrize("dt", DT_IDS)
@pytest.mark.parametrize("case", HALF_BWD, ids=dc.case_id)
def test_half_backward_is_the_fp32_backward_on_the_up_cast_operands(pvb, case, dt):
    assert dp.vec(case) and case.dg > 1
    half_backward_check(pvb, case, "random", dt)


GRID_CALLS = [(case, layout, dt) for dt in DT_IDS for case in dp.PATHS for layout in dp.LAYOUTS]


def profile_grid_calls(trace):
    """Runs the half-precision forward of every GRID_CALLS entry under torch.profiler and writes its trace to `trace`."""
    import clean_pvnet_b200 as pvb
    ops = [lowp(dc.make_inputs(case, seed=1, offsets="random"), DTYPES[dt]) for case, _, dt in GRID_CALLS]
    for (case, layout, _), o in zip(GRID_CALLS, ops):     # module load and first launches outside the profile
        run(pvb, case, *o, layout)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for (case, layout, _), o in zip(GRID_CALLS, ops):
            run(pvb, case, *o, layout)
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)


def test_each_forward_launches_the_grid_the_twin_computes(tmp_path):
    """The profiler's record of every half-precision forward launch of PATHS, both layouts and dtypes: grid
    (ceil(P / 64) * S, ceil(C_out / 128), B), with S the twin's half_splits.  The profile runs in a child process and
    leaves no profiler state in this one: after a profiling session in a process, a later session there can miss a
    kernel's record, which the kernel count of test_gpu_dcn_nhwc.py's copy test would see."""
    trace = tmp_path / "trace.json"
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    path = [root, os.path.join(root, "oracle"), here, os.environ.get("PYTHONPATH", "")]
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(trace)], capture_output=True, text=True,
                       env=dict(os.environ, PYTHONPATH=os.pathsep.join(p for p in path if p)), timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel" and
                      ("dcn_forward_half_kernel" in e["name"] or "dcn_forward_nhwc_kernel" in e["name"])),
                     key=lambda e: e["ts"])
    assert [("nhwc" in e["name"], tuple(e["args"]["grid"])) for e in kernels] == \
        [(layout == "channels_last", dp.grid(case)) for case, layout, _ in GRID_CALLS]


if __name__ == "__main__":
    profile_grid_calls(sys.argv[1])
