#!/usr/bin/env python
"""Build the UNMODIFIED reference deformable PSROI pooling kernels (lib/csrc/dcn_v2/src/cuda/
dcn_v2_psroi_pooling_cuda.cu) into oracle/_ref/libdcn_pool_ref.so.

TEST INFRASTRUCTURE ONLY.  Nothing under `oracle/` is imported by the product package (`clean_pvnet_b200/`).

The file's host functions are written against ATen / THC and do not build on current torch, but everything before the
first of them -- bilinear_interp and the two kernel templates -- uses nothing from those headers.  So the recipe copies
the file to a scratch directory, keeps it up to the line before `dcn_v2_psroi_pooling_cuda_forward`'s return type, and
appends two `extern "C"` launchers of its own (LAUNCHERS below) with the reference's launch shape: block 512, grid
min(ceil(n / 512), 4096), `top_count` and both gradients zeroed by the caller as the host functions do
(dcn_v2_psroi_pooling_cuda.cu:272-419).  It is compiled with the flags oracle/build_dcn_ref.py uses, for sm_90a,
against the empty stand-ins under oracle/dcn_shim/.  The sources never enter this repository; the output lands in
oracle/_ref/, which git ignores.

Usage:  python oracle/build_dcn_pool_ref.py [--force]      (no-op if the reference checkout is absent)
"""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libdcn_pool_ref.so")
REF = os.environ.get("PVNET_REFERENCE", "/root/reference")
SRC = os.path.join(REF, "lib", "csrc", "dcn_v2", "src", "cuda", "dcn_v2_psroi_pooling_cuda.cu")
FIRST_HOST = "dcn_v2_psroi_pooling_cuda_forward("

# torch.utils.cpp_extension's CUDAExtension nvcc flags, plus setup.py's define_macros / extra_compile_args["nvcc"]
FLAGS = ["-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_BFLOAT16_CONVERSIONS__",
         "-D__CUDA_NO_HALF2_OPERATORS__", "--expt-relaxed-constexpr", "-std=c++17",
         "-DWITH_CUDA", "-DCUDA_HAS_FP16=1",
         "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
         "-Xcompiler", "-fPIC", "--shared", "-cudart", "static"]

# Written here, not taken from the reference: the host functions' launches with raw pointers (P = pooled_height =
# pooled_width, as the host functions pass).  The caller zeroes count, grad_input and grad_trans.
LAUNCHERS = r'''
static dim3 ref_grid(int n) { return dim3(std::min((n + 511) / 512, 4096)); }

extern "C" void ref_dcn_pool_forward(const float *input, const float *rois, const float *trans, float *out,
                                     float *count, int n_roi, int C, int H, int W, int P, int part_size,
                                     int sample_per_part, int num_classes, int no_trans, float spatial_scale,
                                     float trans_std, cudaStream_t s)
{
    const int n = n_roi * C * P * P;
    if (n == 0) return;
    DeformablePSROIPoolForwardKernel<float><<<ref_grid(n), 512, 0, s>>>(
        n, input, spatial_scale, C, H, W, P, P, rois, trans, no_trans, trans_std, sample_per_part, C, 1, part_size,
        num_classes, C / num_classes, out, count);
}

extern "C" void ref_dcn_pool_backward(const float *grad_out, const float *count, const float *input, const float *rois,
                                      const float *trans, float *grad_input, float *grad_trans, int n_roi, int C,
                                      int H, int W, int P, int part_size, int sample_per_part, int num_classes,
                                      int no_trans, float spatial_scale, float trans_std, cudaStream_t s)
{
    const int n = n_roi * C * P * P;
    if (n == 0) return;
    DeformablePSROIPoolBackwardAccKernel<float><<<ref_grid(n), 512, 0, s>>>(
        n, grad_out, count, n_roi, spatial_scale, C, H, W, P, P, C, grad_input, grad_trans, input, rois, trans,
        no_trans, trans_std, sample_per_part, 1, part_size, num_classes, C / num_classes);
}
'''


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def build(force=False):
    if not os.path.exists(SRC):
        print(f"[build_dcn_pool_ref] {SRC} not present; nothing to do (a prebuilt oracle/_ref/libdcn_pool_ref.so is used "
              "as-is)")
        return False
    if os.path.exists(LIB) and not force:
        print(f"[build_dcn_pool_ref] up to date: {LIB}")
        return True
    lines = open(SRC).read().splitlines(keepends=True)
    cut = next(i for i, line in enumerate(lines) if line.startswith(FIRST_HOST))
    while cut > 0 and not lines[cut - 1].strip() == "":      # drop the return type line(s) above the name
        cut -= 1
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="pvnet_dcn_pool_ref_build_")
    try:
        src = os.path.join(tmp, "dcn_v2_psroi_pooling_kernels.cu")
        with open(src, "w") as fh:
            fh.write("".join(lines[:cut]) + LAUNCHERS)
        out = os.path.join(tmp, "libdcn_pool_ref.so")
        subprocess.check_call([_nvcc(), src, "-I", tmp, "-I", os.path.join(HERE, "dcn_shim")] + FLAGS + ["-o", out],
                              cwd=tmp)
        shutil.copy(out, LIB)
        print(f"[build_dcn_pool_ref] built {LIB}")
        return True
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
