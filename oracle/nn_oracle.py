"""ctypes front-end of the nearest-neighbour oracle (oracle/nn_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of nn_oracle.c.  Imported by tests/; never by the product package.
"""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "nn_oracle.c")
_SO = os.path.join(_HERE, "libnn_oracle.so")
_LIB = None

# the flags of oracle/Makefile: no fusions the source does not spell out, no fast math
_CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra"]


def _has_fma():
    try:
        with open("/proc/cpuinfo") as fh:
            return re.search(r"\bfma\b", fh.read()) is not None
    except OSError:
        return False


def build(force=False):
    if force or not os.path.exists(_SO) or os.path.getmtime(_SRC) > os.path.getmtime(_SO):
        cc = os.environ.get("CC") or shutil.which("gcc") or "cc"
        flags = _CFLAGS + (["-mfma"] if _has_fma() else [])
        subprocess.check_call([cc] + flags + ["-shared", "-o", _SO, _SRC, "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = ctypes.CDLL(_SO)
        _LIB.orc_nearest_point_idx.restype = None
        _LIB.orc_nearest_point_idx.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 5
    return _LIB


def nearest_point_idx(ref, que, exclude_self=False):
    """findNearestPointIdxLauncher (lib/csrc/nn/src/nearest_neighborhood.cu:123-163) on the CPU: ref [b,pn1,dim],
    que [b,pn2,dim] (rounded to float32), dim 2 or 3 -> int32 [b,pn2]."""
    ref = np.ascontiguousarray(ref, np.float32)
    que = np.ascontiguousarray(que, np.float32)
    b, pn1, dim = ref.shape
    assert que.shape[0] == b and que.shape[2] == dim and dim in (2, 3)
    pn2 = que.shape[1]
    idxs = np.zeros((b, pn2), dtype=np.int32)
    lib().orc_nearest_point_idx(ref.ctypes.data, que.ctypes.data, idxs.ctypes.data, b, pn1, pn2, dim,
                                int(bool(exclude_self)))
    return idxs
