#!/usr/bin/env python
"""Build the UNMODIFIED reference nearest-neighbour extension (lib/csrc/nn) into oracle/_ref/libnn_ref.so.

TEST INFRASTRUCTURE ONLY.  Nothing under `oracle/` is imported by the product package (`clean_pvnet_b200/`).

The reference's recipe (lib/csrc/nn/setup.py) is `nvcc src/nearest_neighborhood.cu -c -x cu -Xcompiler -fPIC -O2
-arch=sm_52`, linked by cffi against libcudart.  Its launcher `findNearestPointIdxLauncher` is already `extern "C"` and
takes host pointers, so this compiles the same source with the same flags straight into a shared library that ctypes
loads; no cffi module is built.  On an H100 the driver JIT-compiles the embedded compute_52 PTX, exactly what a
reference user running on that GPU gets.  The source is copied to a scratch directory (the reference tree is read-only
and its sources never enter this repository); the output lands in oracle/_ref/, which git ignores.

Usage:  python oracle/build_nn_ref.py [--force]      (no-op if the reference checkout is absent)
"""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libnn_ref.so")
REF = os.environ.get("PVNET_REFERENCE", "/root/reference")
SRC = os.path.join(REF, "lib", "csrc", "nn", "src", "nearest_neighborhood.cu")


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def build(force=False):
    if not os.path.exists(SRC):
        print(f"[build_nn_ref] {SRC} not present; nothing to do (a prebuilt oracle/_ref/libnn_ref.so is used as-is)")
        return False
    if os.path.exists(LIB) and not force:
        print(f"[build_nn_ref] up to date: {LIB}")
        return True
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="pvnet_nn_ref_build_")
    try:
        src = os.path.join(tmp, "nearest_neighborhood.cu")
        shutil.copy(SRC, src)
        out = os.path.join(tmp, "libnn_ref.so")
        # setup.py's flags (-x cu -Xcompiler -fPIC -O2 -arch=sm_52), linked into one shared object
        subprocess.check_call([_nvcc(), src, "-x", "cu", "-Xcompiler", "-fPIC", "-O2", "-arch=sm_52",
                               "-Wno-deprecated-gpu-targets", "--shared", "-o", out], cwd=tmp)
        shutil.copy(out, LIB)
        print(f"[build_nn_ref] built {LIB}")
        return True
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
