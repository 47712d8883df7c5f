#!/usr/bin/env python
"""Why is a step slower at 8 ranks than at 1?  Runs the bench's timed loop several times per rank under torchrun with
the suspects switched on/off (NVML clock sampler, stage-profiling events, the exchange) and prints, per variant, the
max-over-ranks ms/step, the host time spent enqueueing one step, and every rank's select-stage time.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29521 tools/scale_diag.py
"""
import ctypes
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import clean_pvnet_b200 as pvb
from clean_pvnet_b200 import _lib, parallel, synth
import bench

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
lib = _lib.load()
B, K, HN = 16, 9, 512
mask, vertex, _ = synth.make_inputs("cfg2", device=dev, seed=1236 + rank)
layer = parallel.ShardedVotingLayer(B * world, K, depth=4, device=dev) if world > 1 else None
STEPS = 60


def loop(exchange, sampler_period, profile, reasons_every=1, clock=True):
    def step(i):
        if exchange and layer is not None:
            return layer(mask, vertex, HN, inlier_thresh=0.99, seed=1000 + i)
        return pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=0.99, seed=1000 + i, img_base=rank * B)
    for i in range(5):
        step(i)
    if layer is not None:
        layer.drain()
    torch.cuda.synchronize()
    smp = bench.ClockSampler(local, period=sampler_period, reasons_every=reasons_every, clock=clock) if sampler_period else None
    lib.pvb_profile_reset()
    lib.pvb_profile_enable(1 if profile else 0)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    if smp:
        smp.start()
    # its own event pair, not devtime.device_ms: the window also holds the host clock around the enqueue and the
    # exchange's drain, and the clock sampler starts between the synchronise and the first event
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t0 = time.perf_counter()
    for i in range(STEPS):
        step(i)
    t1 = time.perf_counter()
    if layer is not None:
        layer.drain()
    e1.record()
    torch.cuda.synchronize()
    if smp:
        smp.stop()
    st = (ctypes.c_double * 4)()
    n = lib.pvb_profile_read(st, 4) if profile else 0
    lib.pvb_profile_enable(0)
    vals = torch.tensor([e0.elapsed_time(e1) / STEPS, (t1 - t0) * 1e3 / STEPS, (st[0] / n) if n else 0.0, (st[2] / n) if n else 0.0],
                        dtype=torch.float64, device=dev)
    allv = [torch.zeros_like(vals) for _ in range(world)]
    if world > 1:
        dist.all_gather(allv, vals)
    else:
        allv = [vals]
    return torch.stack(allv).cpu()


variants = [("exchange + sampler 10ms + profile (bench default)", True, 0.01, True),
            ("exchange + profile, no sampler", True, 0, True),
            ("exchange + sampler 10ms, no profile", True, 0.01, False),
            ("exchange only", True, 0, False),
            ("plain v3 (no exchange), nothing else", False, 0, False),
            ("plain v3 + profile", False, 0, True),
            ("exchange + sampler 100ms + profile", True, 0.1, True),
            ("plain v3 + sampler 10ms (clock + reasons)", False, 0.01, False),
            ("plain v3 + sampler 10ms, clock only", False, 0.01, False, 10 ** 9, True),
            ("plain v3 + sampler 10ms, reasons only", False, 0.01, False, 1, False),
            ("plain v3 + sampler 2ms (clock + reasons)", False, 0.002, False)]
for v in variants:
    name, ex, per, prof = v[:4]
    r = loop(ex, per, prof, *v[4:])
    if rank == 0:
        print(f"{name:52s} ms/step max {r[:, 0].max():.4f} (rank0 {r[0, 0]:.4f})  host enqueue ms/step max {r[:, 1].max():.4f}  "
              f"select us per rank {[round(float(x) * 1e3, 1) for x in r[:, 2]]}  vote us rank0 {float(r[0, 3]) * 1e3:.1f}", flush=True)
if rank == 0:
    print("usable cores:", bench._usable_cores(), "cpu_count:", os.cpu_count())
if world > 1:
    dist.barrier()
    if layer is not None:
        layer.close()
    dist.destroy_process_group()
