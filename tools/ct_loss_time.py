#!/usr/bin/env python
"""Times the CenterNet detector's heatmap loss on the device two ways, at the detector's training output (128x104) and
validation output (184x136), with B = 4 (the reference's default batch) and B = 32, C = 30 and 20 objects per image,
using CUDA events after warm-up:
  reference  the dense float32 ct_hm [B,30,H,W] copied host-to-device from pinned memory, then the trainer's expression
             (net_utils.FocalLoss on net_utils.sigmoid, lib/train/trainers/ct.py:20) forward, and forward + backward
  fused      clean_pvnet_b200.ct_focal_loss forward, and forward + backward, from the [B,M] objects
It also prints the fused kernels' HBM traffic (logits read twice, grad written once) over the data sheet's 3.35 TB/s as
a lower bound on their time, and the bytes per batch each form sends through the loader.  Prints the card, its power
limit and SM clock beside the numbers."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from devtime import card_line, device_ms  # noqa: E402

HBM_BPS = 3.35e12
C, M = 30, 20
REPS, WARMUP = 50, 5           # per timing: calls in the event window, calls before it


def focal_loss(logits, gt):
    """net_utils.FocalLoss()(net_utils.sigmoid(logits), gt), as the reference trainer runs it."""
    pred = torch.clamp(logits.sigmoid(), min=1e-4, max=1 - 1e-4)
    pos_inds = gt.eq(1).float()
    neg_inds = gt.lt(1).float()
    neg_weights = torch.pow(1 - gt, 4)
    pos_loss = (torch.log(pred) * torch.pow(1 - pred, 2) * pos_inds).sum()
    neg_loss = (torch.log(1 - pred) * torch.pow(pred, 2) * neg_weights * neg_inds).sum()
    num_pos = pos_inds.float().sum()
    if num_pos == 0:
        return 0 - neg_loss
    return 0 - (pos_loss + neg_loss) / num_pos


def objects(B, H, W, seed):
    """M objects per image with radii like the detector's boxes produce (up to 31 at 128x104, 42 at 184x136)."""
    rng = np.random.default_rng(seed)
    ind = torch.from_numpy(rng.integers(0, H * W, (B, M)).astype(np.int64))
    rad = torch.from_numpy(rng.integers(0, max(H, W) // 4 + 1, (B, M)).astype(np.int32))
    cls = torch.from_numpy(rng.integers(0, C, (B, M)).astype(np.int64))
    c01 = torch.ones(B, M)
    return ind, rad, cls, c01


def run(B, H, W):
    dev = torch.device("cuda", 0)
    objs_h = objects(B, H, W, seed=H + B)
    objs = [t.to(dev) for t in objs_h]
    dense_d = pvb.ct_target_batch(*objs, C, H, W)
    dense_h = dense_d.cpu().pin_memory()
    x = torch.randn(B, C, H, W, device=dev).requires_grad_()
    got = torch.autograd.grad(pvb.ct_focal_loss(x, *objs), x)[0]
    want = torch.autograd.grad(focal_loss(x, dense_d), x)[0]
    r = {"B": B, "C": C, "H": H, "W": W, "M": M, "grad_bit_equal": bool(torch.equal(got, want)),
         "loss_fused": float(pvb.ct_focal_loss(x.detach(), *objs)), "loss_torch": float(focal_loss(x.detach(), dense_d))}
    r["ref_h2d_ms"] = device_ms(lambda: dense_d.copy_(dense_h, non_blocking=True), REPS, WARMUP)
    r["ref_fwd_ms"] = device_ms(lambda: focal_loss(x.detach(), dense_d), REPS, WARMUP)
    r["ref_fwd_bwd_ms"] = device_ms(lambda: torch.autograd.grad(focal_loss(x, dense_d), x), REPS, WARMUP)
    r["fused_fwd_ms"] = device_ms(lambda: pvb.ct_focal_loss(x.detach(), *objs), REPS, WARMUP)
    r["fused_fwd_bwd_ms"] = device_ms(lambda: torch.autograd.grad(pvb.ct_focal_loss(x, *objs), x), REPS, WARMUP)
    r["target_kernel_ms"] = device_ms(lambda: pvb.ct_target_batch(*objs, C, H, W), REPS, WARMUP)
    n = B * C * H * W
    r["fused_fwd_hbm_bytes"] = 4 * n
    r["fused_fwd_bwd_hbm_bytes"] = 3 * 4 * n
    r["fused_fwd_bwd_hbm_bound_ms"] = 3 * 4 * n / HBM_BPS * 1e3
    r["loader_bytes_dense"] = int(dense_h.numel() * 4)
    r["loader_bytes_objects"] = int(sum(t.numel() * t.element_size() for t in objs_h))
    return r


def main():
    assert torch.cuda.is_available(), "ct_loss_time.py measures on a CUDA device"
    print(f"card: {card_line()}  torch {torch.__version__}")
    for H, W in ((104, 128), (136, 184)):
        for B in (4, 32):
            r = run(B, H, W)
            print(json.dumps(r))
            print(f"  B={B} {W}x{H}: H2D dense {r['ref_h2d_ms']:.3f} ms | torch fwd {r['ref_fwd_ms']:.3f}, fwd+bwd "
                  f"{r['ref_fwd_bwd_ms']:.3f} ms | fused fwd {r['fused_fwd_ms']:.3f}, fwd+bwd {r['fused_fwd_bwd_ms']:.3f}"
                  f" ms (HBM bound {r['fused_fwd_bwd_hbm_bound_ms']:.3f}) | target kernel {r['target_kernel_ms']:.3f} ms"
                  f" | loader bytes {r['loader_bytes_dense']} vs {r['loader_bytes_objects']}"
                  f" | grad bit-equal {r['grad_bit_equal']}")


if __name__ == "__main__":
    main()
