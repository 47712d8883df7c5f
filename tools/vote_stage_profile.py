#!/usr/bin/env python
"""Per-kernel times of the bench step (ransac_voting_layer_v3, hn = 512, t = 0.99, bench.py's inputs), in a process of
its own: 20 warm-up steps, then 30 steps under torch.profiler with CUDA activities.  Prints one table row per launch
position of the step: the kernel (demangled name without its parameter list), its mean time and the mean gap before it.
The GPU's name, power limit and max SM clock are read in the same run.

For the pruned vote it also prints, per pass, the inlier tests the lists asked for (sum over (image, keypoint) of list
length x selected pixels, counted by re-running the profiled steps' seeds unprofiled) and the tests per second that
gives with that pass's mean kernel time; for the full vote kernel (--full, or wherever pruning does not run) hn x pixels.

    python tools/vote_stage_profile.py [--workload cfg2|cfg4] [--full] [--out FILE.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from clean_pvnet_b200 import _lib, synth, ransac_voting_gpu as rv  # noqa: E402

HN, THRESH = 512, 0.99          # bench.py's step
WARMUP, STEPS = 20, 30


def _smi(field):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader,nounits", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def _kernel_name(name):
    name = re.sub(r"^void\s+", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):      # drop the parameter list, keep the template arguments
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return name[:cut]


def _pass_tests(mask, vertex, step, debug):
    """inlier tests per pass, [pass 1, pass 2], of the step with this seed (None when the call did not prune)"""
    pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=1000 + step, debug=debug)
    torch.cuda.synchronize()
    lib = _lib.load()
    m, v = rv._check_inputs(mask, vertex)
    d = rv._make_desc(m, v, HN, THRESH, 5, 30000, _lib.PVB_SELECT_BYTE, 1000 + step, 0, None)
    ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
    L = _lib.PvbLayout()
    _lib.check(lib.pvb_workspace_layout(d, L))
    B, K = d.B, d.K
    tn = np.minimum(ws[L.tn:L.tn + 4 * B].view(torch.int32).cpu().numpy(), L.capacity).astype(np.int64)
    if debug:
        return [float(tn.sum() * K * HN)]
    lens = ws[L.prune_len:L.prune_len + 2 * B * K * 4].view(torch.int32).view(2, B, K).cpu().numpy().astype(np.int64)
    return [float((lens[p] * tn[:, None]).sum()) for p in range(2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=["cfg2", "cfg4"])
    ap.add_argument("--full", action="store_true", help="score every hypothesis (debug=True): the full vote kernel")
    ap.add_argument("--out", default=None, help="also write the result as JSON")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vote_stage_profile.py needs a CUDA device (there is no CPU path to time)")
    dev = torch.device("cuda", 0)
    mask, vertex, _ = synth.make_inputs(args.workload, device=dev, seed=1234 + 2)
    B, K = vertex.shape[0], vertex.shape[3]

    def step(i):
        return pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=1000 + i, debug=args.full)

    for i in range(WARMUP):
        step(i)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(STEPS):
            step(i)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                  key=lambda e: e.time_range.start)
    if len(kern) % STEPS:
        raise SystemExit(f"{len(kern)} device activities do not split into {STEPS} equal steps")
    per = len(kern) // STEPS
    rows = []
    for j in range(per):
        evs = [kern[s * per + j] for s in range(STEPS)]
        names = {_kernel_name(e.name) for e in evs}
        if len(names) != 1:
            raise SystemExit(f"launch {j} of the step is not one kernel: {sorted(names)}")
        dur = np.mean([e.time_range.end - e.time_range.start for e in evs])
        gap = np.mean([e.time_range.start - kern[s * per + j - 1].time_range.end for s, e in enumerate(evs)]) if j else 0.0
        rows.append(dict(launch=j, kernel=names.pop(), us=float(dur), gap_before_us=float(gap)))

    pruned = not args.full and any("prune_hist_kernel" in r["kernel"] for r in rows)
    tests = np.mean([_pass_tests(mask, vertex, i, not pruned) for i in range(STEPS)], axis=0)
    votes = [r for r in rows if re.search(r"vote(_list)?_kernel", r["kernel"])]
    for r, t in zip(votes, tests):
        r["tests"] = float(t)
        r["tests_per_s"] = float(t / (r["us"] * 1e-6))
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=_smi("power.limit"), sm_clock_max_mhz=_smi("clocks.max.sm"),
               workload=args.workload, B=B, K=K, hn=HN, thresh=THRESH, pruned=pruned, warmup=WARMUP, steps=STEPS,
               kernels=rows)
    if pruned:
        first = next(r for r in rows if "prune_hist_kernel" in r["kernel"])
        last = votes[-1]
        res["vote_stage_us"] = float(sum(r["us"] + r["gap_before_us"] for r in rows[first["launch"]:last["launch"] + 1])
                                     - first["gap_before_us"])
    print(f"{res['gpu']}, power limit {res['power_limit_w']} W, max SM clock {res['sm_clock_max_mhz']} MHz; "
          f"{args.workload} (B={B}, K={K}, hn={HN}, t={THRESH}), {'full' if not pruned else 'pruned'} vote, "
          f"mean of {STEPS} steps after {WARMUP} warm-up steps")
    print(f"{'#':>2}  {'kernel':<58} {'us':>8} {'gap':>6} {'tests':>10} {'T tests/s':>9}")
    for r in rows:
        t = f"{r['tests'] / 1e6:9.1f}M {r['tests_per_s'] / 1e12:9.2f}" if "tests" in r else ""
        print(f"{r['launch']:>2}  {r['kernel'][:58]:<58} {r['us']:8.1f} {r['gap_before_us']:6.1f} {t}")
    if pruned:
        print(f"vote stage (prune_hist_kernel .. last vote kernel, gaps included): {res['vote_stage_us']:.1f} us")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
