"""Builds libpvnet_vote_b200.so (hand-written sm_90a CUDA for the H100 behind a C ABI) in-tree with nvcc.

    python clean_pvnet_b200/build.py [--force] [--verbose]

The .so is a build product (git-ignored).  No JIT,
no torch headers: the library's only dependency is the (statically linked) CUDA runtime.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["api.cu", "select.cu", "vote.cu", "prune.cu", "compat.cu", "pnp.cu", "exchange.cu", "nn.cu", "loss.cu"]
# every header a translation unit includes (pnp.cu: pnp_core.cuh, p3p_core.cuh), found by globbing
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + [os.path.join("..", "..", "include", "pvnet_vote_b200.h")]
LIB = os.path.join(HERE, "libpvnet_vote_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-O2",
    "-Xptxas", "-v",
    "--shared", "-cudart", "static",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    env = dict(os.environ)
    env.pop("CC", None); env.pop("CXX", None)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    if verbose or r.returncode != 0:
        print(r.stdout)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libpvnet_vote_b200.so")
    with open(os.path.join(HERE, "build.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + r.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or True))
