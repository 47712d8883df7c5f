"""Times the CenterNet decode (DESIGN.md 8j) with CUDA events after warm-up, and reads the card's name, power limit
and max SM clock in the same run:
  - the restated torch Network.decode_detection (tests/ct_decode_cases.py) against decode_detections, per call, at
    (B, C, H x W) in {(1, 1, 136x184), (1, 30, 136x184), (16, 1, 136x184), (32, 30, 104x128)};
  - the batched decode_detections -> detection_boxes -> crop_inputs chain at B = 16 against 16 calls of the
    host-syncing cascade path (torch decode of one image, then crop.cascade_crop with its box copy to the host);
  - the one-read byte bound of the logits at 3.35 TB/s, labelled as a bound.

    python tools/ct_decode_time.py [--iters N] [--json out.json]
"""
import argparse
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import clean_pvnet_b200 as pvb  # noqa: E402
import crop_cases as cc  # noqa: E402
import ct_decode_cases as dc  # noqa: E402
from devtime import card_line, device_ms  # noqa: E402

SHAPES = [(1, 1, (136, 184)), (1, 30, (136, 184)), (16, 1, (136, 184)), (32, 30, (104, 128))]


def stand_in_res():
    """lib.networks.ct_pvnet.res for cascade_crop, with get_affine_transform / affine_transform restated."""
    du = types.SimpleNamespace(get_affine_transform=lambda c, s, rot, size, inv=0: cc.crop_matrices(
        c, np.float32(s[0] if np.ndim(s) else s), *size)[inv], affine_transform=cc.dot_affine)
    res = types.ModuleType("lib.networks.ct_pvnet.res")
    res.data_utils = du
    res.tless_config = types.SimpleNamespace(scale_ratio=2.4, mean=cc.MEAN.reshape(1, 1, 3), std=cc.STD.reshape(1, 1, 3))
    res.tless_pvnet_utils = types.SimpleNamespace(input_scale=np.array([256, 256]))
    sys.modules["lib.networks.ct_pvnet.res"] = res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    out = {"card": card_line(), "decode": [], "chain": None}
    print("card:", out["card"])
    rng = np.random.default_rng(0)
    for B, C, hw in SHAPES:
        lg = torch.from_numpy(dc.blobs(rng, B, C, *hw, noise=0.3)).cuda()
        wh = torch.from_numpy(dc._wh(rng, B, *hw)).cuda()
        t_torch = device_ms(lambda: dc.restate_decode(lg, wh, 100), args.iters, 20) * 1e3
        t_fused = device_ms(lambda: pvb.decode_detections(lg, wh), args.iters, 20) * 1e3
        bound = lg.numel() * 4 / 3.35e12 * 1e6
        row = {"B": B, "C": C, "H": hw[0], "W": hw[1], "torch_us": round(t_torch, 2), "fused_us": round(t_fused, 2),
               "logit_read_bound_us": round(bound, 3)}
        out["decode"].append(row)
        print(json.dumps(row))

    stand_in_res()
    B, hw = 16, (136, 184)
    imgs = torch.from_numpy(np.stack([cc.random_images(rng, 1)[0] for _ in range(B)])).cuda()
    lg = torch.from_numpy(dc.blobs(rng, B, 30, *hw, noise=0.3)).cuda()
    wh = torch.from_numpy(dc._wh(rng, B, *hw)).cuda()
    meta_c = torch.tensor([[360.0, 270.0]]).repeat(B, 1)
    meta_s = torch.tensor([[720.0, 720.0]]).repeat(B, 1)
    inp0 = torch.zeros((1, 3, 544, 736))

    def chain():
        _, det = pvb.decode_detections(lg, wh)
        boxes = pvb.detection_boxes(det, meta_c, meta_s, (736, 544))[:, 0]
        return pvb.crop.crop_device(imgs, boxes, torch.arange(B, device="cuda"), (256, 256), 2.4, 0.0, False, True,
                                    False, cc.MEAN.reshape(3), cc.STD.reshape(3))[0]

    def per_image():
        for b in range(B):
            _, det = dc.restate_decode(lg[b:b + 1], wh[b:b + 1], 100)
            batch = {'meta': {'center': meta_c[b:b + 1], 'scale': meta_s[b:b + 1]}, 'inp': inp0}
            pvb.crop.cascade_crop(imgs[b:b + 1], None, batch, {'detection': det})

    out["chain"] = {"B": B, "C": 30, "batched_us": round(device_ms(chain, max(20, args.iters // 4), 20) * 1e3, 1),
                    "per_image_host_sync_us": round(device_ms(per_image, max(5, args.iters // 20), 3) * 1e3, 1)}
    print(json.dumps(out["chain"]))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
