#!/usr/bin/env python
"""Times the evaluator metrics on the device in one process, beside the evaluator's own numpy lines on the same inputs,
and prints a table and one JSON object:

  pose   pvb_pose_metrics (projection_2d + cm_degree_5 distances) for n pose pairs x pn model points, CUDA events after
         warm-up; against lib/evaluators/linemod/pvnet.py:59-66 + :84-94 (two `project` calls, the norm and the mean, and
         cm_degree_5) looped over the n pairs in numpy, host clock
  mask   pvb_mask_iou (its two output memsets and the kernel) on an int64 prediction and a uint8 ground truth of B x 480 x
         640, CUDA events; against linemod/pvnet.py:96-100 per image: the `.cpu()` of both masks (the argmax mask_iou
         recomputes is not counted) and the two numpy passes, host clock.  The rate is set against the data sheet's HBM
         bound (3.35 TB/s on an H100 SXM): B * H * W * 9 bytes read.  The timed calls cycle through enough copies of the
         inputs (>= 200 MB) that they are not served from the 50 MB L2.

The model sizes pn are ASSUMPTIONS spanning a plausible range: the LINEMOD vertex counts are not in this repository.

    python tools/metrics_time.py [--reps N] [--json PATH]
"""
import argparse
import ctypes
import itertools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from devtime import card, card_line, device_ms, host_ms  # noqa: E402

PAIRS = (1, 64, 1024)
SIZES = (1000, 5000, 20000)          # assumed model vertex counts (see above)
MASK_BATCHES = (1, 16)
H, W = 480, 640
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet; a bound, not an expectation
K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])


def _device_us(fn, reps):
    """devtime.device_ms of fn(i), 5 warm-up calls: i counts 0..4 over the warm-up, then again 0..reps-1 over the
    timed calls, so the timed calls start from the first input copy."""
    i = itertools.chain(range(5), range(reps))
    return device_ms(lambda: fn(next(i)), reps, 5) * 1e3


def _poses(rng, n):
    q, _ = np.linalg.qr(rng.normal(size=(n, 3, 3)))
    t = rng.normal(size=(n, 3, 1)) * 0.05 + [[0], [0], [1.0]]
    return np.concatenate([q, t], 2)


def _project(model, K, pose):
    xyz = np.dot(model, pose[:, :3].T) + pose[:, 3:].T
    xyz = np.dot(xyz, K.T)
    return xyz[:, :2] / xyz[:, 2:]


def _numpy_pose(model, pred, gt):
    """linemod/pvnet.py:59-66 and :84-94 for every pair, thresholds included."""
    for p, g in zip(pred, gt):
        np.mean(np.linalg.norm(_project(model, K, p) - _project(model, K, g), axis=-1)) < 5
        t = np.linalg.norm(p[:, 3] - g[:, 3]) * 100
        tr = np.trace(np.dot(p[:, :3], g[:, :3].T))
        tr = tr if tr <= 3 else 3
        tr = tr if tr >= -1 else -1
        t < 5 and np.rad2deg(np.arccos((tr - 1.0) / 2.0)) < 5


def _numpy_mask(pred, gt):
    """linemod/pvnet.py:96-100 per image, with the copies of both masks to the host."""
    for b in range(pred.shape[0]):
        p = pred[b].detach().cpu().numpy()
        g = gt[b].detach().cpu().numpy()
        (p & g).sum() / (p | g).sum() > 0.7


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the JSON object here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("metrics_time.py needs a CUDA device (there is no CPU path to time)")
    lib = pvb._lib.load()
    dev = torch.device("cuda", 0)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    cd = card()
    res = dict(gpu=cd["name"], power_limit_w=cd["power_limit_w"], sm_clock_max_mhz=cd["sm_clock_max_mhz"],
               sizes_are_assumptions=True, pose=[], mask=[])
    rng = np.random.default_rng(0)
    lines = [f"GPU: {card_line(cd)}", "",
             "pvb_pose_metrics          device (us)   numpy loop (us)   speed-up"]
    for pn in SIZES:
        model_h = rng.normal(size=(pn, 3)) * [0.05, 0.03, 0.04]
        model = torch.from_numpy(model_h).to(dev)
        km = torch.from_numpy(K).to(dev)
        for n in PAIRS:
            pred_h, gt_h = _poses(rng, n), _poses(rng, n)
            pp, pg = torch.from_numpy(pred_h).to(dev), torch.from_numpy(gt_h).to(dev)
            outs = [torch.empty(n, dtype=torch.float64, device=dev) for _ in range(3)]
            nb = lib.pvb_pose_metrics_workspace_bytes(n, pn)
            ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
            us = _device_us(lambda i: pvb._lib.check(lib.pvb_pose_metrics(
                model.data_ptr(), pp.data_ptr(), pg.data_ptr(), km.data_ptr(), 0, outs[0].data_ptr(), outs[1].data_ptr(),
                outs[2].data_ptr(), n, pn, ws.data_ptr(), nb, stream)), args.reps)
            np_us = host_ms(lambda: _numpy_pose(model_h, pred_h, gt_h), warmup=1, min_s=0.2) * 1e3
            res["pose"].append(dict(n=n, pn=pn, device_us=us, numpy_us=np_us))
            lines.append(f"  n={n:5d} pn={pn:6d}   {us:12.1f}   {np_us:15.0f}   {np_us / us:8.0f}x")
    lines += ["", "pvb_mask_iou (int64 pred, uint8 gt, 480x640)   device (us)   GB/s   of 3.35 TB/s   numpy + .cpu() (us)"]
    for B in MASK_BATCHES:
        nbytes = B * H * W * 9
        copies = max(2, -(-200_000_000 // nbytes))
        g = torch.Generator(device=dev).manual_seed(B)
        preds = [torch.randint(0, 2, (B, H, W), generator=g, device=dev, dtype=torch.int64) for _ in range(copies)]
        gts = [torch.randint(0, 2, (B, H, W), generator=g, device=dev, dtype=torch.uint8) for _ in range(copies)]
        inter = torch.empty(B, dtype=torch.int64, device=dev)
        uni = torch.empty(B, dtype=torch.int64, device=dev)
        st = (ctypes.c_int64 * 3)(H * W, W, 1)
        us = _device_us(lambda i: pvb._lib.check(lib.pvb_mask_iou(
            preds[i % copies].data_ptr(), pvb._lib.PVB_MASK_I64, st, gts[i % copies].data_ptr(), pvb._lib.PVB_MASK_U8, st,
            inter.data_ptr(), uni.data_ptr(), B, H, W, stream)), args.reps)
        p0, g0 = preds[(args.reps - 1) % copies].cpu().numpy(), gts[(args.reps - 1) % copies].cpu().numpy()
        assert inter.tolist() == [int((p0[b] & g0[b]).sum()) for b in range(B)]
        assert uni.tolist() == [int((p0[b] | g0[b]).sum()) for b in range(B)]
        np_us = host_ms(lambda: _numpy_mask(preds[0], gts[0]), warmup=1, min_s=0.2) * 1e3
        rate = nbytes / (us * 1e-6)
        res["mask"].append(dict(B=B, bytes=nbytes, device_us=us, bytes_per_s=rate, fraction_of_hbm_datasheet=rate /
                                HBM_BYTES_PER_S, hbm_bound_us=nbytes / HBM_BYTES_PER_S * 1e6, numpy_with_copies_us=np_us))
        lines.append(f"  B={B:3d} ({nbytes / 1e6:5.1f} MB)                  {us:12.1f}   {rate / 1e9:5.0f}   "
                     f"{rate / HBM_BYTES_PER_S:11.0%}   {np_us:18.0f}")
    print("\n".join(lines))
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
