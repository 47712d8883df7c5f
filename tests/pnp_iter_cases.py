"""Synthetic problems for PVNet's default pose step (`cv2.solvePnP(..., SOLVEPNP_ITERATIVE)`, csrc/pnp_iter_core.cuh),
shared by the CPU pin, the golden-fixture generator and the GPU tests; plus the host build of the core and the reference
call it is pinned to."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_LINEMOD = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])
PNS = (6, 7, 9, 17, 33, 64)
NOISES = (0.0, 1.0, 5.0, 20.0)
STATUS = {"ok": 0, "iteration_limit": 1, "too_few_points": 2, "planar": 3, "degenerate": 4}


def _rotation(aa):
    theta = np.linalg.norm(aa)
    if theta == 0:
        return np.eye(3)
    w = aa / theta
    W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    return np.eye(3) + np.sin(theta) * W + (1 - np.cos(theta)) * (W @ W)


def iter_case(seed, pn=9, noise=1.0):
    """One problem: (pts2d [pn,2], pts3d [pn,3], K [3,3]), float64.  The model is pn points of a LINEMOD-sized solid (within
    +-10 cm, never planar), the object 0.3-3 m away; the seed also picks the rotation (generic, within 1e-3 rad of 0, or
    within 1e-7 rad of pi), the intrinsics (LINEMOD's, or scaled and shifted per problem) and one or two vote outliers
    (keypoints moved by 50-200 px) on top of Gaussian pixel noise."""
    rng = np.random.default_rng(seed)
    pts3d = rng.uniform(-0.1, 0.1, (pn, 3)) * rng.uniform(0.3, 1.0, 3)
    kind = seed % 5
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    if kind == 3:
        aa = axis * rng.uniform(0, 1e-3)
    elif kind == 4:
        aa = axis * (np.pi - rng.uniform(0, 1e-7))
    else:
        aa = axis * rng.uniform(0.1, 3.0)
    depth = float(np.exp(rng.uniform(np.log(0.3), np.log(3.0))))
    t = np.array([rng.uniform(-0.1, 0.1) * depth, rng.uniform(-0.08, 0.08) * depth, depth])
    K = K_LINEMOD.copy()
    if rng.uniform() < 0.5:
        K[:2, :2] *= rng.uniform(0.8, 1.2)
        K[:2, 2] += rng.uniform(-20, 20, 2)
    cam = pts3d @ _rotation(aa).T + t
    uv = np.stack([K[0, 0] * cam[:, 0] / cam[:, 2] + K[0, 2], K[1, 1] * cam[:, 1] / cam[:, 2] + K[1, 2]], 1)
    uv += rng.normal(size=uv.shape) * noise
    for i in rng.choice(pn, int(rng.integers(0, 3)), replace=False):
        d = rng.normal(size=2)
        uv[i] += d / np.linalg.norm(d) * rng.uniform(50, 200)
    return uv, pts3d, K


def cases(count, seed0=0):
    """`count` problems cycling over pn in PNS and noise in NOISES"""
    return [iter_case(seed0 + s, PNS[s % len(PNS)], NOISES[(s // len(PNS)) % len(NOISES)]) for s in range(count)]


def opencv_pnp(pts3d, pts2d, K):
    """(rvec, tvec) of cv2.solvePnP called as lib/utils/pvnet/pvnet_pose_utils.py:5-38 calls it (zero distortion)"""
    import cv2
    _, r, t = cv2.solvePnP(np.ascontiguousarray(pts3d, np.float64), np.ascontiguousarray(pts2d, np.float64),
                           np.asarray(K, np.float64), np.zeros(shape=[8, 1], dtype="float64"), flags=cv2.SOLVEPNP_ITERATIVE)
    return np.concatenate([r.ravel(), t.ravel()])


def rel_diff(a, b):
    """max |a - b| over max(1, max |a|): the pin's measure on (rvec, tvec) (relative for metre-scale translations, absolute
    for small rotation vectors)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(1.0, float(np.abs(a).max())))


def host_core():
    """The host build of csrc/pnp_iter_core.cuh (tests/pnp_iter_host_harness.cpp, g++): solve(pts2d [n,pn,2], pts3d [pn,3] |
    [n,pn,3], K [3,3] | [n,3,3]) -> (pose [n,3,4], rt [n,6], info [n,2])."""
    out = os.path.join(ROOT, "tests", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libpnp_iter_host.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-x", "c++",
                           os.path.join(ROOT, "tests", "pnp_iter_host_harness.cpp"), "-o", so])
    lib = ctypes.CDLL(so)
    DP = ctypes.POINTER(ctypes.c_double)

    def ptr(a):
        return a.ctypes.data_as(DP)

    def solve(pts2d, pts3d, K):
        p2 = np.ascontiguousarray(pts2d, np.float64)
        p3 = np.ascontiguousarray(pts3d, np.float64)
        km = np.ascontiguousarray(K, np.float64)
        n, pn = p2.shape[:2]
        pose, rt = np.zeros((n, 3, 4)), np.zeros((n, 6))
        info = np.zeros((n, 2), np.int32)
        lib.pnp_iter_host_solve(ptr(p2), ptr(p3), ptr(km), ptr(pose), ptr(rt),
                                info.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), ctypes.c_int(n), ctypes.c_int(pn),
                                ctypes.c_longlong(0 if p3.ndim == 2 else pn * 3), ctypes.c_longlong(0 if km.ndim == 2 else 9))
        return pose, rt, info

    def rodrigues(r):
        R, J = np.zeros(9), np.zeros(27)
        lib.pnp_iter_host_rodrigues(ptr(np.ascontiguousarray(r, np.float64)), ptr(R), ptr(J))
        return R.reshape(3, 3), J.reshape(3, 9)

    def rotation_to_vector(R):
        r = np.zeros(3)
        lib.pnp_iter_host_rotation_to_vector(ptr(np.ascontiguousarray(R, np.float64)), ptr(r))
        return r

    solve.rodrigues = rodrigues
    solve.rotation_to_vector = rotation_to_vector
    return solve
