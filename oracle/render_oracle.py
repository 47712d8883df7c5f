"""ctypes front-end of the depth-renderer oracle (oracle/render_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of render_oracle.c.  Imported by tests/; never by the product package.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "render_oracle.c")
_SO = os.path.join(_HERE, "librender_oracle.so")
_LIB = None

# the flags of oracle/Makefile: no fusions the source does not spell out, no fast math
_CFLAGS = ["-O2", "-fPIC", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra"]


def build(force=False):
    if force or not os.path.exists(_SO) or os.path.getmtime(_SRC) > os.path.getmtime(_SO):
        cc = os.environ.get("CC") or shutil.which("gcc") or "cc"
        subprocess.check_call([cc] + _CFLAGS + ["-shared", "-o", _SO, _SRC, "-lm"])
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = ctypes.CDLL(_SO)
        _LIB.orc_render_depth.restype = None
        _LIB.orc_render_depth.argtypes = ([ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double]
                                          + [ctypes.c_void_p] * 4)
    return _LIB


def render_depth(pts, faces, pose, K, size, near=100.0, far=10000.0):
    """One pose: pts [V,3], faces [F,3], pose [3,4] ([R|t]), K [3,3], size (W, H).  The points and the pose are rounded to
    float32 first, as the device renderer rounds them.  Returns dict(z=, edge=, gap=, clip=), each float64 [H,W]
    (see render_oracle.c)."""
    pts = np.ascontiguousarray(pts, np.float32)
    faces = np.ascontiguousarray(faces, np.int32)
    pose = np.ascontiguousarray(np.asarray(pose, np.float64).astype(np.float32), np.float64)
    K = np.ascontiguousarray(K, np.float64)
    W, H = size
    out = {k: np.zeros((H, W), np.float64) for k in ("z", "edge", "gap", "clip")}
    lib().orc_render_depth(pts.ctypes.data, pts.shape[0], faces.ctypes.data, faces.shape[0], pose.ctypes.data,
                           K.ctypes.data, H, W, float(near), float(far), out["z"].ctypes.data, out["edge"].ctypes.data,
                           out["gap"].ctypes.data, out["clip"].ctypes.data)
    return out
