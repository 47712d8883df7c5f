#!/usr/bin/env python
"""Times the nearest-neighbour port in one process and prints one JSON object:

  reference   the reference launcher findNearestPointIdxLauncher (oracle/_ref/libnn_ref.so, built unmodified by
              oracle/build_nn_ref.py) on host arrays: the host wall clock per call, which is what nn_utils costs a user
              (three cudaMalloc, three copies in, one out, three cudaFree, kernel; skipped where it was not built)
  device      pvb_nearest_point_idx on device-resident fp32 points (CUDA events, after warm-up)
  add_metric  pvb_add_metric, ADD-S and ADD, for batches of 1 and 64 pose pairs (CUDA events)

for model sizes pn in {1 000, 5 000, 20 000} (ref = que = pn points).  The vertex counts of the LINEMOD and T-LESS models
are not part of this repository: these sizes are ASSUMPTIONS spanning a plausible range, not the datasets' own.
The rate is set against an ESTIMATE of the FP32 issue bound, not a measurement: 9 FP32-pipe instructions per tested pair
(3 FADD, FMUL, 2 FFMA, FSETP and two selects, read from the SASS of the 3-D kernel) at 128 lanes per SM per clock.

    python tools/nn_time.py [--reps N]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402

SIZES = (1000, 5000, 20000)        # assumed model vertex counts (see above)
BATCHES = (1, 64)
INSTR_PER_PAIR = 9                 # estimate from SASS, see above
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libnn_ref.so")


def _smi(field):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={field}", "--format=csv,noheader,nounits", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def _events_us(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def _poses(rng, n):
    q, _ = np.linalg.qr(rng.normal(size=(n, 3, 3)))
    t = rng.normal(size=(n, 3, 1)) * 0.1 + [[0], [0], [1.0]]
    return np.concatenate([q, t], 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    clouds = {pn: (rng.normal(size=(1, pn, 3)) * 0.05).astype(np.float32) for pn in SIZES}
    queries = {pn: (clouds[pn] + rng.normal(size=(1, pn, 3)).astype(np.float32) * 1e-3).astype(np.float32) for pn in SIZES}
    poses = {n: (_poses(rng, n), _poses(rng, n)) for n in BATCHES}
    if not torch.cuda.is_available():
        raise SystemExit("nn_time.py needs a CUDA device (there is no CPU path to time)")
    lib = pvb._lib.load()
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    sm_clock_mhz = _smi("clocks.max.sm")
    bound = props.multi_processor_count * 128 * sm_clock_mhz * 1e6 / INSTR_PER_PAIR if sm_clock_mhz else None
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    ref_lib = None
    if os.path.exists(REF_LIB):
        ref_lib = ctypes.CDLL(REF_LIB)
        ref_lib.findNearestPointIdxLauncher.restype = None
        ref_lib.findNearestPointIdxLauncher.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 5
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit_w=_smi("power.limit"), sm_clock_max_mhz=sm_clock_mhz,
               sms=props.multi_processor_count, sizes_are_assumptions=True,
               fp32_issue_bound_estimate_pairs_per_s=bound, rows=[])
    for pn in SIZES:
        row = dict(pn=pn, pairs=pn * pn)
        r_h, q_h = clouds[pn], queries[pn]
        if ref_lib is not None:
            idx_h = np.zeros((1, pn), np.int32)
            call = lambda: ref_lib.findNearestPointIdxLauncher(r_h.ctypes.data, q_h.ctypes.data, idx_h.ctypes.data,  # noqa: E731
                                                               1, pn, pn, 3, 0)
            for _ in range(3):
                call()                                   # the first call JIT-compiles the reference's compute_52 PTX
            t0 = time.perf_counter()
            for _ in range(args.reps):
                call()
            row["reference_host_us"] = (time.perf_counter() - t0) / args.reps * 1e6
        r, q = torch.from_numpy(r_h).to(dev), torch.from_numpy(q_h).to(dev)
        idx = torch.empty((1, pn), dtype=torch.int32, device=dev)
        nb = lib.pvb_nearest_point_workspace_bytes(1, pn, pn)
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
        us = _events_us(lambda: pvb._lib.check(lib.pvb_nearest_point_idx(r.data_ptr(), q.data_ptr(), idx.data_ptr(), 1, pn, pn,
                                                                         3, 0, ws.data_ptr(), nb, stream)), args.reps)
        row["device_us"] = us
        row["device_pairs_per_s"] = pn * pn / (us * 1e-6)
        if ref_lib is not None:
            assert np.array_equal(idx.cpu().numpy(), idx_h)
        model = torch.from_numpy(r_h[0].astype(np.float64)).to(dev)
        for n in BATCHES:
            pp, pg = (torch.from_numpy(p).to(dev) for p in poses[n])
            out = torch.empty(n, dtype=torch.float64, device=dev)
            for syn in (1, 0):
                nb = lib.pvb_add_metric_workspace_bytes(n, pn, syn)
                w = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
                us = _events_us(lambda: pvb._lib.check(lib.pvb_add_metric(model.data_ptr(), pp.data_ptr(), pg.data_ptr(),
                                                                          out.data_ptr(), n, pn, syn, w.data_ptr(), nb,
                                                                          stream)), args.reps)
                key = f"add{'s' if syn else ''}_n{n}"
                row[key + "_us"] = us
                if syn:
                    row[key + "_pairs_per_s"] = n * pn * pn / (us * 1e-6)
        if bound:
            row["device_fraction_of_bound"] = row["device_pairs_per_s"] / bound
            row["adds_n64_fraction_of_bound"] = row["adds_n64_pairs_per_s"] / bound
        res["rows"].append(row)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
