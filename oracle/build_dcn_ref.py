#!/usr/bin/env python
"""Build the UNMODIFIED reference DCNv2 sampling kernels (lib/csrc/dcn_v2/src/cuda/dcn_v2_im2col_cuda.cu) into
oracle/_ref/libdcn_ref.so.

TEST INFRASTRUCTURE ONLY.  Nothing under `oracle/` is imported by the product package (`clean_pvnet_b200/`).

The reference extension as a whole cannot be built against current torch (dcn_v2_cuda.cu is written against THC), but
its three launchers -- modulated_deformable_im2col_cuda, modulated_deformable_col2im_cuda and
modulated_deformable_col2im_coord_cuda -- live in dcn_v2_im2col_cuda.cu, are already `extern "C"`, take device pointers
and a stream, and use nothing from the ATen / THC headers that file includes.  So the file and its header are copied
to a scratch directory and compiled with the nvcc defines torch's CUDAExtension and the reference's setup.py pass, for
sm_90a, against the empty stand-ins under oracle/dcn_shim/.  ctypes calls the launchers directly; the tests restate
the reference's GEMM steps (dcn_v2_cuda.cu) themselves.  The sources never enter this repository; the output lands in
oracle/_ref/, which git ignores.

Usage:  python oracle/build_dcn_ref.py [--force]      (no-op if the reference checkout is absent)
"""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libdcn_ref.so")
REF = os.environ.get("PVNET_REFERENCE", "/root/reference")
SRC = os.path.join(REF, "lib", "csrc", "dcn_v2", "src", "cuda")
FILES = ["dcn_v2_im2col_cuda.cu", "dcn_v2_im2col_cuda.h"]

# torch.utils.cpp_extension's CUDAExtension nvcc flags, plus setup.py's define_macros / extra_compile_args["nvcc"]
FLAGS = ["-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_BFLOAT16_CONVERSIONS__",
         "-D__CUDA_NO_HALF2_OPERATORS__", "--expt-relaxed-constexpr", "-std=c++17",
         "-DWITH_CUDA", "-DCUDA_HAS_FP16=1",
         "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
         "-Xcompiler", "-fPIC", "--shared", "-cudart", "static"]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def build(force=False):
    if not all(os.path.exists(os.path.join(SRC, f)) for f in FILES):
        print(f"[build_dcn_ref] {SRC} not present; nothing to do (a prebuilt oracle/_ref/libdcn_ref.so is used as-is)")
        return False
    if os.path.exists(LIB) and not force:
        print(f"[build_dcn_ref] up to date: {LIB}")
        return True
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="pvnet_dcn_ref_build_")
    try:
        for f in FILES:
            shutil.copy(os.path.join(SRC, f), os.path.join(tmp, f))
        out = os.path.join(tmp, "libdcn_ref.so")
        subprocess.check_call([_nvcc(), os.path.join(tmp, FILES[0]), "-I", tmp, "-I", os.path.join(HERE, "dcn_shim")]
                              + FLAGS + ["-o", out], cwd=tmp)
        shutil.copy(out, LIB)
        print(f"[build_dcn_ref] built {LIB}")
        return True
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
