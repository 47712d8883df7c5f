#!/usr/bin/env python
"""Times the v3 step (bench.py's call: hn = 512, t = 0.99, a new seed every step, one caller stream) for each grouped-launch
setting of pvb_set_group_tuning(max_groups, streams) (DESIGN.md 4.4).  The settings are interleaved over --reps rounds
so that clock drift hits them alike; prints the median and range of ms per step of each.

    python tools/group_sweep.py [--workload cfg2|cfg4] [--settings 1x1 2x2 4x2 ...] [--steps 200] [--reps 3]
"""
import argparse
import itertools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=["cfg2", "cfg4"])
    ap.add_argument("--settings", nargs="+", default=["1x1", "2x2", "4x2", "4x3", "4x4", "8x2", "8x4"],
                    help="GROUPSxSTREAMS")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    import clean_pvnet_b200 as pvb
    from clean_pvnet_b200 import _lib, synth
    from devtime import card_line, device_ms
    if not torch.cuda.is_available():
        raise SystemExit("group_sweep.py needs a CUDA device")
    lib = _lib.load()
    mask, vertex, _ = synth.make_inputs(args.workload, device="cuda:0", seed=1236)
    settings = [tuple(int(x) for x in s.split("x")) for s in args.settings]
    times = {s: [] for s in settings}
    for rep in range(args.reps):
        for g, s in settings:
            _lib.check(lib.pvb_set_group_tuning(g, s))
            seeds = itertools.chain(range(10), range(1000, 1000 + args.steps))      # warm-up seeds, then timed ones
            times[(g, s)].append(device_ms(lambda: pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99,
                                                                              seed=next(seeds)), args.steps, 10))
    _lib.check(lib.pvb_set_group_tuning(0, 0))
    print(f"{args.workload} on {card_line()}: ms per step, median [min, max] of {args.reps}")
    for (g, s), t in times.items():
        t = sorted(t)
        print(f"  groups <= {g:2d}, streams {s}: {t[len(t) // 2]:.4f} [{t[0]:.4f}, {t[-1]:.4f}]")


if __name__ == "__main__":
    main()
