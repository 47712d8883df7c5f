"""Times T-LESS's PVNet crop (DESIGN.md 8g): the device crop_inputs (CUDA events) against the reference's per-box host
path -- cv2.warpAffine + the box mask + the normalisation of pvnet_transform, then the host-to-device copy of each input
as the cascade makes it -- for n boxes from 720x540 images at both T-LESS input sizes.  One JSON line per case; with
--out FILE.json the whole result is also written there.

    python tools/crop_time.py [--reps 50] [--out crop_time.json]

The written bytes (the fp32 inputs) over the data sheet's 3.35 TB/s HBM3 rate give a lower bound on the kernel time; it
is labelled a bound, not a measurement.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clean_pvnet_b200 as pvb  # noqa: E402
import crop_cases as cc  # noqa: E402
from devtime import card_line, device_ms, host_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def host_path(imgs, boxes, index, size, scale_ratio, box_ratio):
    import cv2
    w, h = size
    out = []
    for b, i in zip(boxes, index):
        c, s = cc.center_scale(b, scale_ratio)
        src, dst = cc.crop_points(c, s, w, h)
        M = cv2.getAffineTransform(src, dst)
        u8 = cv2.warpAffine(imgs[i], M, (w, h), flags=cv2.INTER_LINEAR)
        p = M[:, :2] @ np.asarray(b, np.float64).reshape(2, 2).T + M[:, 2:]
        mean = p.mean(axis=1, keepdims=True)
        r = np.round((p - mean) * box_ratio + mean).astype(np.int32)
        x0, x1 = np.clip(r[0], 0, w - 1)
        y0, y1 = np.clip(r[1], 0, h - 1)
        keep = np.zeros_like(u8)
        keep[y0:y1 + 1, x0:x1 + 1] = u8[y0:y1 + 1, x0:x1 + 1]
        inp = cc.normalise(keep)
        out.append(torch.from_numpy(np.ascontiguousarray(inp)).cuda()[None])
    torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("crop_time needs a CUDA device")
    rng = np.random.default_rng(2026)
    imgs_h = cc.random_images(rng, 4)
    imgs = torch.from_numpy(imgs_h).cuda()
    info = card_line()
    results = []
    for size, scale_ratio, box_ratio in cc.CONFIGS.values():
        for n in (1, 16, 256):
            boxes = cc.random_boxes(rng, n)
            index = rng.integers(0, len(imgs_h), n)
            bd = torch.from_numpy(boxes).cuda()
            ix = torch.from_numpy(index).cuda()
            dev_ms = device_ms(lambda: pvb.crop_inputs(imgs, bd, ix, size, scale_ratio, box_ratio), args.reps, 5)
            host_path(imgs_h, boxes[:1], index[:1], size, scale_ratio, box_ratio)      # warm cv2 and the copy path
            host = host_ms(lambda: host_path(imgs_h, boxes, index, size, scale_ratio, box_ratio),
                           reps=max(1, min(args.reps, 2000 // n)), warmup=0)
            written = n * 3 * size[0] * size[1] * 4
            r = {"gpu": info, "input": f"{size[0]}x{size[1]}", "n": n, "device_ms": round(dev_ms, 4),
                 "host_per_box_path_ms": round(host, 3), "speedup": round(host / dev_ms, 1),
                 "written_bytes": written, "write_bound_ms": round(written / HBM_BYTES_PER_S * 1e3, 4),
                 "write_bound_share": round(written / HBM_BYTES_PER_S * 1e3 / dev_ms, 3)}
            print(json.dumps(r), flush=True)
            results.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
