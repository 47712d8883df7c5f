#!/usr/bin/env python
"""Shows how a grouped v3 step overlaps (DESIGN.md 4.4): bench.py's cfg-2 call (hn = 512, t = 0.99), 20 warm-up steps,
then 10 steps under torch.profiler with CUDA activities.  From the kernel records of the trace (name, stream, start,
duration) it prints, per kernel: launches per step, mean duration, and the share of its time during which pass 1 of the
vote (vote_kernel) of another group ran on another stream.  The GPU's name and power limit are read in the same run.

    python tools/group_overlap.py [--workload cfg2|cfg4] [--groups G --streams S] [--trace FILE.json]
"""
import argparse
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HN, THRESH = 512, 0.99
WARMUP, STEPS = 20, 10


def _short(name):
    name = re.sub(r"^void\s+", "", name)
    name = name.split("(")[0]
    return re.sub(r"^pvb::", "", re.sub(r"<.*", "", name))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=["cfg2", "cfg4"])
    ap.add_argument("--groups", type=int, default=0, help="pvb_set_group_tuning max_groups (0: default)")
    ap.add_argument("--streams", type=int, default=0, help="pvb_set_group_tuning streams (0: default)")
    ap.add_argument("--trace", default=None, help="also keep the Chrome trace here")
    args = ap.parse_args()
    import torch
    import clean_pvnet_b200 as pvb
    from clean_pvnet_b200 import _lib, synth
    from devtime import card_line
    if not torch.cuda.is_available():
        raise SystemExit("group_overlap.py needs a CUDA device")
    lib = _lib.load()
    _lib.check(lib.pvb_set_group_tuning(args.groups, args.streams))
    mask, vertex, _ = synth.make_inputs(args.workload, device="cuda:0", seed=1236)
    for i in range(WARMUP):
        pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=i)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(STEPS):
            pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=1000 + i)
        torch.cuda.synchronize()
    path = args.trace or os.path.join(tempfile.mkdtemp(), "trace.json")
    prof.export_chrome_trace(path)
    _lib.check(lib.pvb_set_group_tuning(0, 0))
    with open(path) as fh:
        evs = json.load(fh)["traceEvents"]
    kern = [(_short(e["name"]), e["tid"], float(e["ts"]), float(e["ts"]) + float(e["dur"]))
            for e in evs if e.get("cat") == "kernel"]
    pass1 = [k for k in kern if k[0] == "vote_kernel"]
    stats = {}
    for name, tid, t0, t1 in kern:
        under = 0.0
        if name != "vote_kernel":
            iv = sorted((max(t0, a0), min(t1, a1)) for _, s, a0, a1 in pass1 if s != tid and a0 < t1 and a1 > t0)
            end = t0
            for a, b in iv:             # union of the intervals
                a = max(a, end)
                if b > a:
                    under += b - a
                    end = b
        s = stats.setdefault(name, [0, 0.0, 0.0])
        s[0] += 1; s[1] += t1 - t0; s[2] += under
    span = (max(k[3] for k in kern) - min(k[2] for k in kern)) / STEPS
    print(f"{card_line()}; {args.workload}, groups <= {args.groups or 'default'}, streams {args.streams or 'default'}; "
          f"{STEPS} profiled steps, {span:.1f} us of kernels per step (first start to last end)")
    print(f"{'kernel':<28} {'per step':>8} {'mean us':>8} {'under pass 1':>13}")
    first = {}
    for name, _, t0, _ in kern:
        first.setdefault(name, t0)
    for name, (n, dur, under) in sorted(stats.items(), key=lambda x: first[x[0]]):
        print(f"{name[:28]:<28} {n / STEPS:8.1f} {dur / n:8.1f} {(under / dur if dur else 0):12.0%}")


if __name__ == "__main__":
    main()
