#!/usr/bin/env python
"""Times ransac_voting_layer_v3 stage by stage (pvb_profile_*) for vote-kernel launch shapes."""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from clean_pvnet_b200 import _lib, synth  # noqa: E402
from devtime import device_ms  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--cfg", default="cfg2")
ap.add_argument("--hn", type=int, default=512)
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--B", type=int, default=None)
ap.add_argument("--chunks", default="0", help="gather modes (pvb_set_tuning): 0 auto, 1 pixel-wise, 2 row-wise")
ap.add_argument("--variants", default="0,1")
args = ap.parse_args()
lib = _lib.load()
mask, vertex, _ = synth.make_inputs(args.cfg, device="cuda", seed=1236, B=args.B)
ref = None
for variant in [int(v) for v in args.variants.split(",")]:
    for chunk in [int(c) for c in args.chunks.split(",")]:
        _lib.check(lib.pvb_set_tuning(chunk, variant))
        for i in range(5):
            out = pvb.ransac_voting_layer_v3(mask, vertex, args.hn, inlier_thresh=0.99, seed=7)
        if ref is None:
            ref = out.clone()
        same = bool(torch.equal(ref, out))
        torch.cuda.synchronize()
        lib.pvb_profile_reset(); lib.pvb_profile_enable(1)
        seeds = iter(range(100, 100 + args.steps))
        step = device_ms(lambda: pvb.ransac_voting_layer_v3(mask, vertex, args.hn, inlier_thresh=0.99, seed=next(seeds)),
                         args.steps, 0)
        ms = (ctypes.c_double * 4)()
        n = lib.pvb_profile_read(ms, 4)
        lib.pvb_profile_enable(0)
        print(f"variant={variant} gather={chunk} step={step:.4f} ms  "
              f"select={ms[0]/n:.4f} gen={ms[1]/n:.4f} vote={ms[2]/n:.4f} refit={ms[3]/n:.4f}  same_result={same}")
