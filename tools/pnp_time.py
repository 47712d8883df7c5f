#!/usr/bin/env python
"""Times the three batched uncertainty-PnP entries for a few batch sizes (one warp per problem): uncertainty_pnp_batch
(fp64 inputs, LM refinement from a given start), p3p_init_batch (the P3P start alone) and uncertainty_pnp_from_votes (fp32
keypoints and weights, LM refinement from the same start), next to the same arithmetic core compiled for the host
(tests/pnp_host_harness.cpp, one core) on the same problems."""
import ctypes
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from util import pnp_case  # noqa: E402
from devtime import device_ms  # noqa: E402

cases = [pnp_case(1000 + s, pn=9, noise=2.0) for s in range(256)]
so = os.path.join(ROOT, "tests", "_build", "libpnp_host.so")
os.makedirs(os.path.dirname(so), exist_ok=True)
subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-x", "c++", os.path.join(ROOT, "tests", "pnp_host_harness.cpp"), "-o", so])
lib = ctypes.CDLL(so)
DP = ctypes.POINTER(ctypes.c_double)
t0 = time.perf_counter()
out = np.empty(6)
info = (ctypes.c_int * 2)()
for c in cases:
    a = [np.ascontiguousarray(x) for x in c[:5]]
    lib.pnp_host_solve(*[x.ctypes.data_as(DP) for x in a], out.ctypes.data_as(DP), info, ctypes.c_int(9), ctypes.c_int(50),
                       ctypes.c_double(1e-6), ctypes.c_double(1e-10), ctypes.c_double(1e-8))
cpu_us = (time.perf_counter() - t0) / len(cases) * 1e6
print(f"host build of the same core, 1 core: {cpu_us:.1f} us per problem (incl. ctypes call)")


for n in (1, 16, 256, 4096):
    reps = [cases[i % 256] for i in range(n)]
    f = lambda i: torch.from_numpy(np.stack([c[i] for c in reps])).cuda()  # noqa: E731
    uv, p3, W, K, init = f(0), f(1), f(2), f(3), f(4)
    uv32, W32 = uv.float(), W.float()
    _, inf = pvb.uncertainty_pnp_batch(uv, W, p3, K, init, return_info=True)
    t_batch = device_ms(lambda: pvb.uncertainty_pnp_batch(uv, W, p3, K, init), 20, 3) * 1e3
    t_p3p = device_ms(lambda: pvb.p3p_init_batch(uv, W, p3, K), 20, 3) * 1e3
    t_votes = device_ms(lambda: pvb.uncertainty_pnp_from_votes(uv32, None, p3, K, init, weights=W32), 20, 3) * 1e3
    print(f"n={n:5d}: uncertainty_pnp_batch {t_batch:8.1f} us ({t_batch / n:7.2f} us/problem, mean iterations "
          f"{inf[:, 0].float().mean().item():.2f})  p3p_init_batch {t_p3p:8.1f} us  uncertainty_pnp_from_votes {t_votes:8.1f} us")
