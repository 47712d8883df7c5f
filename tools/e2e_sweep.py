#!/usr/bin/env python
"""End-to-end (pinned host tensors in, host keypoints out) timing of the host entry for chunk sizes / modes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import clean_pvnet_b200 as pvb
from clean_pvnet_b200 import synth
from devtime import device_ms

mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=1236)
mh, vh = mask.cpu().pin_memory(), vertex.cpu().pin_memory()
oh = torch.empty((16, 9, 2)).pin_memory()
ref = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99, seed=3).cpu()
for zc in ("auto", "inplace", "staged"):
    for chunk in (1, 2, 4, 8, 16):
        for i in range(3):
            o = pvb.ransac_voting_layer_v3_host(mh, vh, 512, inlier_thresh=0.99, seed=3, chunk_images=chunk, out=oh, mode=zc)
        ok = bool(torch.equal(o, ref))
        seeds = iter(range(100, 120))
        ms = device_ms(lambda: pvb.ransac_voting_layer_v3_host(mh, vh, 512, inlier_thresh=0.99, seed=next(seeds),
                                                               chunk_images=chunk, out=oh, mode=zc), 20, 0)
        print(f"mode={zc} chunk={chunk:2d}  {ms:.3f} ms/step  same_as_device={ok}")
