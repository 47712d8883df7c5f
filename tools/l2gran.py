#!/usr/bin/env python
"""Experiment: does cudaLimitMaxL2FetchGranularity change what the gather kernel pulls from DRAM?

The selected pixels' vertex rows are 72 B at 8-byte alignment, one in ~10 pixels: with 64-byte DRAM fetches a row costs
2 x 64 B on average (1.78x), with 32-byte fetches 3 x 32 B (1.33x).  Run under ncu:
    ncu --cache-control all --metrics dram__bytes_read.sum,gpu__time_duration.sum -k regex:gather python tools/l2gran.py 32
"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import clean_pvnet_b200 as pvb
from clean_pvnet_b200 import _lib, synth
from devtime import device_ms

gran = int(sys.argv[1]) if len(sys.argv) > 1 else 0
torch.cuda.init()
torch.zeros(1, device="cuda")
rt = ctypes.CDLL("libcudart.so.12")
cur = ctypes.c_size_t()
rt.cudaDeviceGetLimit(ctypes.byref(cur), 5)            # cudaLimitMaxL2FetchGranularity = 0x05
print("granularity before:", cur.value)
if gran:
    rc = rt.cudaDeviceSetLimit(5, ctypes.c_size_t(gran))
    rt.cudaDeviceGetLimit(ctypes.byref(cur), 5)
    print("set ->", gran, "rc", rc, "now", cur.value)
mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=1236)
lib = _lib.load()
for i in range(3):
    pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99, seed=i)
torch.cuda.synchronize()
lib.pvb_profile_reset(); lib.pvb_profile_enable(1)
seeds = iter(range(100, 120))
ms = device_ms(lambda: pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99, seed=next(seeds)), 20, 0)
st = (ctypes.c_double * 4)()
n = lib.pvb_profile_read(st, 4)
print(f"gran={cur.value} step {ms:.4f} ms  select {st[0]/n:.4f} generate {st[1]/n:.4f} vote {st[2]/n:.4f} refit {st[3]/n:.4f}")
