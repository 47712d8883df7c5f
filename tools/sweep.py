#!/usr/bin/env python
"""Throughput sweep over the other BASELINE.json configurations (cfg-3, cfg-4, cfg-5 grid) on one GPU.

Prints one markdown table row per case: ms/step (CUDA events, 3 warm-up + N timed), images*keypoints/s, inlier tests/s of
the vote kernel, algorithmic bytes (SURVEY 8d) per second vs the measured HBM peak, stage times.
    python tools/sweep.py [--B 64] [--steps 10] > gpurun_out/sweep.md
"""
import argparse
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from clean_pvnet_b200 import _lib, synth  # noqa: E402
from devtime import device_ms  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=64)
ap.add_argument("--steps", type=int, default=10)
args = ap.parse_args()
lib = _lib.load()
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    peak = 6650.0

cases = [("cfg3 Occlusion-LINEMOD", dict(B=64, H=480, W=640, K=9, hn=1024, fill=(0.05, 0.15), kind="fragmented")),
         ("cfg4 T-LESS share (16 img/GPU)", dict(B=16, H=720, W=540, K=17, hn=512, fill=(0.30, 0.30), kind="blob"))]
for K in (4, 9, 17):
    for hn in (128, 512, 2048):
        for fill in (0.01, 0.30, 0.80):
            cases.append((f"cfg5 K={K} hn={hn} fill={int(fill * 100)}%",
                          dict(B=args.B, H=640, W=640, K=K, hn=hn, fill=(fill, fill), kind="blob")))

print("| case | B | K | hn | mean tn | ms/step | img*kpt/s | vote T tests/s | alg. GB/s (of %.0f) | select / gen / vote / refit ms |" % peak)
print("|---|---|---|---|---|---|---|---|---|---|")
for name, cfg in cases:
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=4242)
    B, H, W, K, hn = cfg["B"], cfg["H"], cfg["W"], cfg["K"], cfg["hn"]
    _, dbg = pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=0.99, seed=1, debug=True)
    tn_sum = int(dbg["tn"].sum().item())
    del dbg
    for i in range(3):
        pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=0.99, seed=2 + i)
    torch.cuda.synchronize()
    lib.pvb_profile_reset(); lib.pvb_profile_enable(1)
    seeds = iter(range(10, 10 + args.steps))
    ms = device_ms(lambda: pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=0.99, seed=next(seeds)), args.steps, 0)
    st = (ctypes.c_double * 4)()
    n = lib.pvb_profile_read(st, 4); lib.pvb_profile_enable(0)
    stage = [st[i] / n for i in range(4)]
    alg = B * H * W * 8 + tn_sum * K * 8 + B * K * 8
    tests = K * hn * tn_sum
    print(f"| {name} | {B} | {K} | {hn} | {tn_sum / B:.0f} | {ms:.3f} | {B * K / ms * 1e3:,.0f} | {tests / stage[2] / 1e9:.2f} | "
          f"{alg / ms / 1e6:.0f} ({100 * alg / ms / 1e6 / peak:.1f} %) | {stage[0]:.3f} / {stage[1]:.3f} / {stage[2]:.3f} / {stage[3]:.3f} |")
    del mask, vertex
    torch.cuda.empty_cache()
