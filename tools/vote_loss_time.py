#!/usr/bin/env python
"""Times PVNet's vote loss on the device two ways, at B = 32, K = 9, 480x640 and 256x256 (the sampler's extreme sizes),
with about 30 % of each mask foreground, using CUDA events after warm-up:
  reference  the dense float32 target [B,2K,H,W] copied host-to-device from pinned memory, then the trainer's expression
             (lib/train/trainers/pvnet.py:25-27) forward and backward in torch
  fused      the keypoints [B,K,2] copied host-to-device from pinned memory, then clean_pvnet_b200.vote_loss forward and
             backward
It also prints the fused kernels' HBM traffic (pred read twice, grad written once, mask read twice) over the data sheet's
3.35 TB/s as a lower bound on their time, the host cost per sample of the target each form needs (the numpy
restatement of compute_vertex, tests/vote_target_cases.py, against the compact keypoint array), and the bytes per batch
each form sends through the loader.  Prints the card, its power limit and SM clock beside the numbers."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from clean_pvnet_b200.vote_loss import compact_vertex  # noqa: E402
from vote_target_cases import restate_vertex  # noqa: E402

HBM_BPS = 3.35e12
B, K = 32, 9


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:        # the numbers below stand without it, but say so
        q = f"(nvidia-smi unavailable: {e})"
    return q


def per_call_ms(fn, reps=30):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def masks(H, W, seed):
    """B masks, each an ellipse covering about 30 % of the image, with the keypoints around it."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    out = np.zeros((B, H, W), np.uint8)
    for b in range(B):
        cx, cy = rng.uniform(0.4, 0.6) * W, rng.uniform(0.4, 0.6) * H
        ax = np.sqrt(0.3 * H * W / np.pi * W / H)
        ay = 0.3 * H * W / np.pi / ax
        out[b] = ((xx - cx) / ax) ** 2 + ((yy - cy) / ay) ** 2 <= 1
    kpt = np.stack([rng.uniform(0.2 * W, 0.8 * W, (B, K)), rng.uniform(0.2 * H, 0.8 * H, (B, K))], -1)
    return out, kpt


def reference_loss(pred, mask, vertex):
    weight = mask[:, None].float()
    vote_loss = F.smooth_l1_loss(pred * weight, vertex * weight, reduction='sum')
    return vote_loss / weight.sum() / vertex.size(1)


def run(H, W):
    dev = torch.device("cuda", 0)
    mask_np, kpt_np = masks(H, W, seed=H)
    t0 = time.perf_counter()
    dense_np = np.stack([restate_vertex(m, k) for m, k in zip(mask_np, kpt_np)])
    host_dense_ms = (time.perf_counter() - t0) / B * 1e3
    t0 = time.perf_counter()
    for _ in range(100):
        compact_np = np.stack([compact_vertex(m, k).transpose(2, 0, 1) for m, k in zip(mask_np, kpt_np)])
    host_compact_ms = (time.perf_counter() - t0) / 100 / B * 1e3
    dense_h = torch.from_numpy(dense_np).pin_memory()
    kpt_h = torch.from_numpy(np.ascontiguousarray(compact_np[:, :, 0, :].transpose(0, 2, 1))).pin_memory()
    mask = torch.from_numpy(mask_np).to(dev)
    pred = torch.randn(B, 2 * K, H, W, device=dev).requires_grad_()
    dense_d = torch.empty_like(dense_h, device=dev)
    kpt_d = torch.empty_like(kpt_h, device=dev)

    def ref_h2d():
        dense_d.copy_(dense_h, non_blocking=True)

    def ref_loss():
        torch.autograd.grad(reference_loss(pred, mask, dense_d), pred)

    def fused_h2d():
        kpt_d.copy_(kpt_h, non_blocking=True)

    def fused_loss():
        torch.autograd.grad(pvb.vote_loss(pred, mask, kpt_d), pred)

    def fused_fwd():
        pvb.vote_loss(pred.detach(), mask, kpt_d)

    ref_h2d()
    fused_h2d()
    torch.cuda.synchronize()
    got = torch.autograd.grad(pvb.vote_loss(pred, mask, kpt_d), pred)[0]
    want = torch.autograd.grad(reference_loss(pred, mask, dense_d), pred)[0]
    r = {"H": H, "W": W, "B": B, "K": K, "fill": float(mask_np.mean()), "grad_bit_equal": bool(torch.equal(got, want))}
    r["ref_h2d_ms"] = per_call_ms(ref_h2d)
    r["ref_fwd_bwd_ms"] = per_call_ms(ref_loss)
    r["ref_total_ms"] = per_call_ms(lambda: (ref_h2d(), ref_loss()))
    r["fused_h2d_ms"] = per_call_ms(fused_h2d)
    r["fused_fwd_ms"] = per_call_ms(fused_fwd)
    r["fused_fwd_bwd_ms"] = per_call_ms(fused_loss)
    r["fused_total_ms"] = per_call_ms(lambda: (fused_h2d(), fused_loss()))
    hbm = (2 * B * 2 * K * H * W * 4) + (B * 2 * K * H * W * 4) + 2 * B * H * W * mask.element_size()
    r["fused_hbm_bytes"] = hbm
    r["fused_hbm_bound_ms"] = hbm / HBM_BPS * 1e3
    r["host_compute_vertex_ms_per_sample"] = host_dense_ms
    r["host_compact_ms_per_sample"] = host_compact_ms
    r["loader_bytes_dense"] = int(dense_np.nbytes)
    r["loader_bytes_compact"] = int(compact_np.nbytes)
    r["loader_bytes_mask"] = int(mask_np.nbytes)
    return r


def main():
    assert torch.cuda.is_available(), "vote_loss_time.py measures on a CUDA device"
    print(f"card: {card()}  torch {torch.__version__}")
    for H, W in ((480, 640), (256, 256)):
        r = run(H, W)
        print(json.dumps(r))
        print(f"  {H}x{W}: reference {r['ref_total_ms']:.3f} ms (H2D {r['ref_h2d_ms']:.3f} + loss {r['ref_fwd_bwd_ms']:.3f})"
              f" | fused {r['fused_total_ms']:.3f} ms (H2D {r['fused_h2d_ms']:.3f} + loss {r['fused_fwd_bwd_ms']:.3f},"
              f" forward alone {r['fused_fwd_ms']:.3f}) | HBM bound {r['fused_hbm_bound_ms']:.3f} ms"
              f" | host per sample {r['host_compute_vertex_ms_per_sample']:.2f} ms vs"
              f" {r['host_compact_ms_per_sample'] * 1e3:.1f} us | loader bytes {r['loader_bytes_dense']} vs"
              f" {r['loader_bytes_compact']}")


if __name__ == "__main__":
    main()
