#!/usr/bin/env python
"""Pass 1 of the pruned v3 vote (vote_kernel<4,128,8,1024,1,...>, DESIGN.md 4.2) on the bench step (hn = 512, t = 0.99,
bench.py's inputs), in a process of its own: its kernel time, and how many of its tests the per-box classification
resolved against how many it scored one hypothesis at a time.  The GPU's name, power limit and max SM clock are read in
the same run.

Kernel time: 20 warm-up steps, then 30 steps under torch.profiler with CUDA activities; the pass-1 launches are picked by
name, so the image groups' overlapping launches need no order.  `--groups 1` (the default) runs every call as one chain on
the caller's stream (pvb_set_group_tuning), so pass 1 runs alone and its time is its own; `--groups 0` keeps the default
grouped step, where pass 1 of one group shares the GPU with the other group's kernels.

Test counts: the same 30 steps again, unprofiled, with pvb_set_pass1_stats set; a library without it (before the per-box
classification) scores every test one by one.

    python tools/pass1_profile.py [--workload cfg2|cfg4] [--groups 1|0] [--out FILE.json]
"""
import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from clean_pvnet_b200 import _lib, synth, ransac_voting_gpu as rv  # noqa: E402
from devtime import card, card_line  # noqa: E402

HN, THRESH = 512, 0.99          # bench.py's step
WARMUP, STEPS = 20, 30
PASS1 = re.compile(r"vote_kernel<4, ?128, ?8, ?1024, ?1(, ?true)?>")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=["cfg2", "cfg4"])
    ap.add_argument("--groups", type=int, default=1, help="1: one chain per call (pass 1 alone); 0: the default groups")
    ap.add_argument("--out", default=None, help="also write the result as JSON")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pass1_profile.py needs a CUDA device (there is no CPU path to time)")
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    _lib.check(lib.pvb_set_group_tuning(args.groups, 0))
    mask, vertex, _ = synth.make_inputs(args.workload, device=dev, seed=1234 + 2)
    B, K = vertex.shape[0], vertex.shape[3]

    def step(i):
        return pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=1000 + i)

    for i in range(WARMUP):
        step(i)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(STEPS):
            step(i)
        torch.cuda.synchronize()
    p1 = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and PASS1.search(e.name)]
    if not p1 or len(p1) % STEPS:
        raise SystemExit(f"{len(p1)} pass-1 launches do not split into {STEPS} steps")
    us = float(sum(e.time_range.end - e.time_range.start for e in p1) / STEPS)

    # the same steps again, unprofiled: pass 1's tests (list length x pixels) and, where the library has them, the per-box
    # counters [resolved as inliers, resolved, scored one by one]
    stats = torch.zeros(3, dtype=torch.int64, device=dev)
    counters = hasattr(lib, "pvb_set_pass1_stats")
    if counters:
        _lib.check(lib.pvb_set_pass1_stats(stats.data_ptr()))
    total = 0
    for i in range(STEPS):
        step(i)
        torch.cuda.synchronize()
        m, v = rv._check_inputs(mask, vertex)
        d = rv._make_desc(m, v, HN, THRESH, 5, 30000, _lib.PVB_SELECT_BYTE, 1000 + i, 0, None)
        ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
        L = _lib.PvbLayout()
        _lib.check(lib.pvb_workspace_layout(d, L))
        tn = np.minimum(ws[L.tn:L.tn + 4 * B].view(torch.int32).cpu().numpy(), L.capacity).astype(np.int64)
        lens = ws[L.prune_len:L.prune_len + B * K * 4].view(torch.int32).view(B, K).cpu().numpy().astype(np.int64)
        total += int((lens * tn[:, None]).sum())
    if counters:
        _lib.check(lib.pvb_set_pass1_stats(None))
    s = stats.cpu().numpy().astype(np.float64) / STEPS
    tests = total / STEPS
    cd = card()
    res = dict(gpu=cd["name"], power_limit_w=cd["power_limit_w"], sm_clock_max_mhz=cd["sm_clock_max_mhz"],
               workload=args.workload, B=B, K=K, hn=HN, thresh=THRESH, groups=args.groups, warmup=WARMUP, steps=STEPS,
               pass1_launches_per_step=len(p1) // STEPS, pass1_us=us, pass1_tests=tests,
               tests_resolved_per_box=float(s[1]) if counters else 0.0,
               tests_resolved_as_inliers=float(s[0]) if counters else 0.0,
               tests_scored=float(s[2]) if counters else tests, per_box_counters=counters)
    print(f"{card_line(cd)}; "
          f"{args.workload} (B={B}, K={K}, hn={HN}, t={THRESH}), groups {args.groups or 'default'}, "
          f"mean of {STEPS} steps after {WARMUP} warm-up steps")
    print(f"pass 1: {us:.1f} us per step in {res['pass1_launches_per_step']} launch(es); {tests / 1e6:.1f} M tests, "
          f"{res['tests_resolved_per_box'] / 1e6:.1f} M resolved per box ({res['tests_resolved_as_inliers'] / 1e6:.1f} M as "
          f"inliers), {res['tests_scored'] / 1e6:.1f} M scored one by one"
          + ("" if counters else " (library without per-box counters: every test scored)"))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
