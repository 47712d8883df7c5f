#!/usr/bin/env python
"""Build the UNMODIFIED reference farthest-point-sampling extension (lib/csrc/fps) into oracle/_ref/libfps_ref.so.

TEST INFRASTRUCTURE ONLY.  Nothing under `oracle/` is imported by the product package (`clean_pvnet_b200/`).

The reference's recipe (lib/csrc/fps/setup.py) is `gcc -shared src/farthest_point_sampling.cpp -c -fopenmp -fPIC -O2
-std=c++11`, linked by cffi with libstdc++.  Its two entries, farthest_point_sampling and
farthest_point_sampling_init_center, are already `extern "C"` and take host pointers, so this compiles the same source
with the same flags into a shared library that ctypes loads; no cffi module is built.  The source is copied to a scratch
directory (the reference tree is read-only and its sources never enter this repository); the output lands in
oracle/_ref/, which git ignores.

Usage:  python oracle/build_fps_ref.py [--force]      (no-op if the reference checkout is absent)
"""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libfps_ref.so")
REF = os.environ.get("PVNET_REFERENCE", "/root/reference")
SRC = os.path.join(REF, "lib", "csrc", "fps", "src", "farthest_point_sampling.cpp")


def build(force=False):
    if not os.path.exists(SRC):
        print(f"[build_fps_ref] {SRC} not present; nothing to do (a prebuilt oracle/_ref/libfps_ref.so is used as-is)")
        return False
    if os.path.exists(LIB) and not force:
        print(f"[build_fps_ref] up to date: {LIB}")
        return True
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="pvnet_fps_ref_build_")
    try:
        src = os.path.join(tmp, "farthest_point_sampling.cpp")
        shutil.copy(SRC, src)
        obj = os.path.join(tmp, "farthest_point_sampling.cpp.o")
        out = os.path.join(tmp, "libfps_ref.so")
        # setup.py's compile line, then the link cffi does (the object plus libstdc++)
        subprocess.check_call(["gcc", "-shared", src, "-c", "-o", obj, "-fopenmp", "-fPIC", "-O2", "-std=c++11"], cwd=tmp)
        subprocess.check_call(["gcc", "-shared", obj, "-o", out, "-lstdc++", "-fopenmp"], cwd=tmp)
        shutil.copy(out, LIB)
        print(f"[build_fps_ref] built {LIB}")
        return True
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
