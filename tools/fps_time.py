#!/usr/bin/env python
"""Times the farthest-point-sampling port in one process and prints one JSON object:

  reference   farthest_point_sampling_init_center of the reference build (oracle/_ref/libfps_ref.so, the unmodified
              lib/csrc/fps source with its setup.py flags) on host arrays: the host wall clock per call, on whatever CPU
              this runs on ("not measured" where the library was not built).  The batch row is the sum of its clouds.
  device      farthest_point_sampling_batch on device-resident points, init_center: CUDA events around `reps` calls
              after warm-up, per call (the host tables' copy and the launch included).

at the shapes (points, keypoints) = (5 000, 8), (100 000, 8), (1 000 000, 8), (100 000, 64), (100 000, 1 024) and a batch
of 30 ragged clouds of 2 000 to 60 000 points at 8 keypoints.  Clouds are seeded Gaussians.  At every shape the device
indices must equal the reference's (or, without the reference build, the numpy restatement's) or the run fails.

    python tools/fps_time.py [--reps N] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
import fps_cases  # noqa: E402
from devtime import card, device_ms  # noqa: E402

SHAPES = ((5000, 8), (100000, 8), (1000000, 8), (100000, 64), (100000, 1024))


def _ref_us(lib, clouds, sn, reps):
    """Median host time of the reference over all clouds, and its indices."""
    times, idxs = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        idxs = [fps_cases.ref_fps(lib, c, sn, 1) for c in clouds]
        times.append(time.perf_counter() - t0)
    return float(np.median(times)) * 1e6, idxs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fps_time.py needs a CUDA device (there is no CPU path to time)")
    dev = torch.device("cuda", 0)
    lib = fps_cases.ref_lib()
    rng = np.random.default_rng(0)
    cd = card()
    res = dict(gpu=cd["name"], power_limit_w=cd["power_limit_w"], sm_clock_max_mhz=cd["sm_clock_max_mhz"],
               reference="libfps_ref.so" if lib is not None else "not measured", rows=[])
    rows = [(f"{pn} points, sn {sn}", [rng.standard_normal((pn, 3)).astype(np.float32)], sn) for pn, sn in SHAPES]
    counts = np.linspace(2000, 60000, 30).astype(np.int32)
    rows.append(("30 ragged clouds, 2000..60000 points, sn 8", [rng.standard_normal((int(c), 3)).astype(np.float32)
                                                                for c in counts], 8))
    for name, clouds, sn in rows:
        n = max(len(c) for c in clouds)
        pad = np.zeros((len(clouds), n, 3), np.float32)
        for b, c in enumerate(clouds):
            pad[b, :len(c)] = c
        x = torch.from_numpy(pad).to(dev)
        cnt = np.array([len(c) for c in clouds], np.int32)
        reps = max(3, min(args.reps, int(2e6 // (n * sn) + 3)))
        us = device_ms(lambda: pvb.farthest_point_sampling_batch(x, sn, counts=cnt), reps, 3) * 1e3
        got = pvb.farthest_point_sampling_batch(x, sn, counts=cnt).cpu().numpy()
        row = dict(shape=name, clouds=len(clouds), points=int(cnt.sum()), sn=sn, device_us=us, device_reps=reps)
        if lib is not None:
            row["reference_host_us"], want = _ref_us(lib, clouds, sn, 3 if n * sn < 1e8 else 1)
            row["speedup"] = row["reference_host_us"] / us
        else:
            row["reference_host_us"] = "not measured"
            want = [fps_cases.fps_restated(c, sn) for c in clouds]
        row["indices_equal"] = all(np.array_equal(got[b], want[b]) for b in range(len(clouds)))
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    if not all(r["indices_equal"] for r in res["rows"]):
        raise SystemExit("device indices differ from the reference")


if __name__ == "__main__":
    main()
