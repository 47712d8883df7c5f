"""Times T-LESS's instance masks on the device (DESIGN.md 8k): instance_masks_batch (render + compose) and the compose
kernel alone (pvb_instance_masks on rendered depth), with CUDA events after a warm-up, at 720 x 540 for B = 16 and 256
images with 1, 8 and 20 instances each, beside the numpy update_mask loop (tests/tless_mask_cases.py's restatement of
handle_test_data.get_mask's compose step) on the same depths on the host.

    python tools/mask_time.py [--out FILE.json]

An icosphere (5 k faces) and a triangle soup (20 k faces) stand in for T-LESS's CAD models, which are not in this
repository.  The OpenGL renderer the reference uses needs a GL context and is not measured here.  The compose kernel's
bound is the bytes it must move (each instance's fp32 depth read once, each int16 label written once) over the H100
SXM data sheet's 3.35 TB/s.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import clean_pvnet_b200 as pvb                         # noqa: E402
from clean_pvnet_b200.render import _compose           # noqa: E402
from tless_mask_cases import compose_restated           # noqa: E402
from vsd_cases import K_TLESS, icosphere, poses, soup   # noqa: E402
from devtime import card_line, device_ms                # noqa: E402

W, H = 720, 540


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON")
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mask_time.py measures on a CUDA device"
    dev = torch.device("cuda", 0)
    meshes = [tuple(torch.from_numpy(a).to(dev) for a in m) for m in (icosphere(4), soup(20_000, extent=60.0))]
    K = torch.from_numpy(K_TLESS).to(dev)
    rows = []
    for B in (16, 256):
        for per in (1, 8, 20):
            n = B * per
            img = np.repeat(np.arange(B), per)
            mi = np.arange(n) % 2
            obj = np.where(mi == 0, 5, 23)
            pz = poses(n, seed=B + per, z=(500.0, 1100.0), xy=120.0)
            pz_dev = torch.from_numpy(pz).to(dev)

            def batch():
                pvb.instance_masks_batch(meshes, mi, obj, img, pz_dev, K, (W, H))
            # the compose step alone, on the depths the batch renders (instance i in slot i)
            depth = torch.empty((n, H, W), dtype=torch.float32, device=dev)
            sels = [torch.from_numpy(np.flatnonzero(mi == k)).to(dev) for k in range(2)]
            for k in range(2):
                depth[sels[k]] = pvb.render_depth_batch(*meshes[k], pz_dev[sels[k]], K, (W, H), 10, 10000)
            pz_mesh = [pz_dev[sels[k]].contiguous() for k in range(2)]

            def render():                                  # the renderer alone, every instance, one launch per mesh
                for k in range(2):
                    pvb.render_depth_batch(*meshes[k], pz_mesh[k], K, (W, H), 10, 10000)
            first = np.searchsorted(img, np.arange(B + 1))
            out = (torch.empty((B, H, W), dtype=torch.int16, device=dev), torch.empty(n, dtype=torch.int64, device=dev),
                   torch.empty(n, dtype=torch.int64, device=dev), torch.empty((n, 4), dtype=torch.int32, device=dev))

            def compose():
                _compose(depth, n, np.arange(n), obj, first, 0, B, H, W, *out, dev)
            for fn in (batch, render, compose):            # one warm-up call each, before any window
                fn()
            t_batch = device_ms(batch, max(2, args.iters // 2), 0)
            t_render = device_ms(render, max(2, args.iters // 2), 0)
            t_compose = device_ms(compose, args.iters, 0)
            # the numpy update_mask loop on the same depths, a few images, per image
            nh = min(B, 4)
            dh = depth[:nh * per].cpu().numpy()
            t0 = time.perf_counter()
            for b in range(nh):
                compose_restated(dh[b * per:(b + 1) * per], obj[b * per:(b + 1) * per])
            t_np = (time.perf_counter() - t0) / nh * 1e3
            bound_ms = (n * H * W * 4 + B * H * W * 2) / 3.35e12 * 1e3
            rows.append(dict(images=B, instances_per_image=per, batch_ms=t_batch, render_ms=t_render, compose_ms=t_compose,
                             compose_hbm_bound_ms=bound_ms, numpy_ms_per_image=t_np, numpy_ms_total=t_np * B,
                             visible_pixels=int(out[2].sum()), rendered_pixels=int(out[1].sum())))
            print(json.dumps(rows[-1]))
    res = dict(gpu=card_line(), size=[W, H], faces=[int(m[1].shape[0]) for m in meshes], rows=rows)
    print(json.dumps(dict(gpu=res["gpu"], faces=res["faces"])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
