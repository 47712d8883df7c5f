#!/usr/bin/env python
"""Times pose.pnp_batch (pvb_pnp_iterative, one warp per problem) for n in {1, 16, 1024} problems of pn = 9 keypoints, with
CUDA events after warm-up, next to a host loop of cv2.solvePnP(..., SOLVEPNP_ITERATIVE) -- what pvnet_pose_utils.pnp runs
per image -- over the same problems.  Prints the card, its power limit and SM clock with the numbers."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from pnp_iter_cases import iter_case, NOISES  # noqa: E402
from devtime import card_line, device_ms, host_ms  # noqa: E402


def main():
    import cv2
    print("card:", card_line())
    cases = [iter_case(50000 + s, 9, NOISES[s % 4]) for s in range(1024)]
    for n in (1, 16, 1024):
        uv = torch.from_numpy(np.stack([c[0] for c in cases[:n]])).cuda()
        X = torch.from_numpy(np.stack([c[1] for c in cases[:n]])).cuda()
        K = torch.from_numpy(np.stack([c[2] for c in cases[:n]])).cuda()
        uv32 = uv.float()
        _, info = pvb.pnp_batch(X, uv, K, return_info=True)
        t_gpu = device_ms(lambda: pvb.pnp_batch(X, uv, K), 50, 5) * 1e3
        t_gpu32 = device_ms(lambda: pvb.pnp_batch(X, uv32, K), 50, 5) * 1e3
        host = [(c[1], c[0], c[2]) for c in cases[:n]]

        def cv_loop():
            for X3, x2, Kc in host:
                cv2.solvePnP(X3, x2, Kc, np.zeros((8, 1)), flags=cv2.SOLVEPNP_ITERATIVE)
        t_cv = host_ms(cv_loop, reps=max(1, 2048 // n), warmup=0) * 1e3
        it = info[:, 0].float()
        print(f"n={n:5d} pn=9: pnp_batch fp64 {t_gpu:8.1f} us, fp32 points {t_gpu32:8.1f} us "
              f"(mean LM iterations {it.mean().item():.2f}, max {int(it.max().item())});  "
              f"cv2.solvePnP loop {t_cv:10.1f} us ({t_cv / n:.1f} us/problem, cv2 {cv2.__version__}, "
              f"{cv2.getNumThreads()} threads)")


if __name__ == "__main__":
    main()
