#!/usr/bin/env python
"""Times pose.pnp_batch (pvb_pnp_iterative, one warp per problem) for n in {1, 16, 1024} problems of pn = 9 keypoints, with
CUDA events after warm-up, next to a host loop of cv2.solvePnP(..., SOLVEPNP_ITERATIVE) -- what pvnet_pose_utils.pnp runs
per image -- over the same problems.  Prints the card, its power limit and SM clock with the numbers."""
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
from pnp_iter_cases import iter_case, NOISES  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:        # the numbers below stand without it, but say so
        q = f"(nvidia-smi unavailable: {e})"
    return q


def per_call_us(fn, reps=50):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def main():
    import cv2
    print("card:", card())
    cases = [iter_case(50000 + s, 9, NOISES[s % 4]) for s in range(1024)]
    for n in (1, 16, 1024):
        uv = torch.from_numpy(np.stack([c[0] for c in cases[:n]])).cuda()
        X = torch.from_numpy(np.stack([c[1] for c in cases[:n]])).cuda()
        K = torch.from_numpy(np.stack([c[2] for c in cases[:n]])).cuda()
        uv32 = uv.float()
        _, info = pvb.pnp_batch(X, uv, K, return_info=True)
        t_gpu = per_call_us(lambda: pvb.pnp_batch(X, uv, K))
        t_gpu32 = per_call_us(lambda: pvb.pnp_batch(X, uv32, K))
        host = [(c[1], c[0], c[2]) for c in cases[:n]]
        reps = max(1, 2048 // n)
        t0 = time.perf_counter()
        for _ in range(reps):
            for X3, x2, Kc in host:
                cv2.solvePnP(X3, x2, Kc, np.zeros((8, 1)), flags=cv2.SOLVEPNP_ITERATIVE)
        t_cv = (time.perf_counter() - t0) / reps * 1e6
        it = info[:, 0].float()
        print(f"n={n:5d} pn=9: pnp_batch fp64 {t_gpu:8.1f} us, fp32 points {t_gpu32:8.1f} us "
              f"(mean LM iterations {it.mean().item():.2f}, max {int(it.max().item())});  "
              f"cv2.solvePnP loop {t_cv:10.1f} us ({t_cv / n:.1f} us/problem, cv2 {cv2.__version__}, "
              f"{cv2.getNumThreads()} threads)")


if __name__ == "__main__":
    main()
