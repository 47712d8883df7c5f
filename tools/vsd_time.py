"""Times T-LESS's VSD on the device (DESIGN.md 8f): the depth rasterizer (pvb_render_depth) and the VSD kernel (pvb_vsd)
separately, with CUDA events after a warm-up, for 16 and 256 pose pairs at 720 x 540 and meshes of about 5 k, 20 k and
100 k faces, beside the numpy VSD restatement of the evaluator on the same host.

    python tools/vsd_time.py [--out FILE.json]

The face counts stand in for T-LESS's CAD models, which are not in this repository.  The OpenGL renderer the reference
uses needs a GL context and is not measured here.  The VSD kernel's bound is the bytes it must read (three fp32 images
per pair) over the H100 SXM data sheet's 3.35 TB/s.
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

import clean_pvnet_b200 as pvb                       # noqa: E402
from clean_pvnet_b200.nn import _call, _workspace   # noqa: E402
from vsd_cases import K_TLESS, icosphere, poses, soup, vsd_restated   # noqa: E402
from devtime import card_line, device_ms                               # noqa: E402

W, H = 720, 540


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "vsd_time.py measures on a CUDA device"
    dev = torch.device("cuda", 0)
    meshes = {"5k": icosphere(4), "20k": icosphere(5), "100k": soup(100_000)}
    rows = []
    for mname, (v, f) in meshes.items():
        pts, faces = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
        for n in (16, 256):
            pe = torch.from_numpy(poses(n, seed=1)).to(dev)
            pg = torch.from_numpy(poses(n, seed=2)).to(dev)
            K = torch.from_numpy(K_TLESS).to(dev)
            B = min(n, 16)
            gt = pvb.render_depth_batch(pts, faces, pg, K, (W, H))
            dt = (gt[:B] + 3.0).contiguous()
            pairs = torch.tensor([(i, i, i % B) for i in range(n)], dtype=torch.int32, device=dev)
            de = pvb.render_depth_batch(pts, faces, pe, K, (W, H))
            e = torch.empty(n, dtype=torch.float64, device=dev)
            nbytes = pvb._lib.load().pvb_vsd_workspace_bytes(n)
            ws = _workspace(nbytes, dev)

            def render():
                pvb.render_depth_batch(pts, faces, pe, K, (W, H))

            def vsd():
                _call("pvb_vsd", dev, dt, B, de, n, 0, gt, n, 0, pairs, n, K, 0, H, W, 15.0, 20.0, e, ws, nbytes)
            for fn in (render, vsd):                       # one warm-up call each, before either window
                fn()
            t_render = device_ms(render, args.iters, 0)
            t_vsd = device_ms(vsd, args.iters, 0)
            t_all = device_ms(lambda: pvb.vsd_batch(pts, faces, pe, pg, K, dt, pairs), max(2, args.iters // 4), 0)
            # numpy restatement of the evaluator's VSD on the same depths, a few pairs, per pair
            de_h, gt_h, dt_h = de[:4].cpu().numpy(), gt[:4].cpu().numpy(), dt[:4].cpu().numpy()
            t0 = time.perf_counter()
            for i in range(4):
                vsd_restated(de_h[i], gt_h[i], dt_h[i], K_TLESS)
            t_np = (time.perf_counter() - t0) / 4 * 1e3
            bound_ms = n * 3 * H * W * 4 / 3.35e12 * 1e3
            rows.append(dict(mesh=mname, faces=int(f.shape[0]), pairs=n, render_ms=t_render, render_ms_per_pose=t_render / n,
                             vsd_ms=t_vsd, vsd_hbm_bound_ms=bound_ms, vsd_batch_ms=t_all, numpy_vsd_ms_per_pair=t_np,
                             numpy_vsd_ms_total=t_np * n))
            print(json.dumps(rows[-1]))
    res = dict(gpu=card_line(), size=[W, H], rows=rows)
    print(json.dumps(dict(gpu=res["gpu"])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
