#!/usr/bin/env python
"""Times DCNv2's TF32 path (csrc/dcn.cu, DESIGN.md section 8p) at the 16 DCN layers of the DLA-34 detector and prints
one JSON object.

Shapes: tests/dcn_cases.DETECTOR at 736x544 (B = 1) and 512x512 (B = 1 and 16), as tools/dcn_time.py.  Per layer and
summed over the 16 layers, in one process on one GPU:

  f32_ieee, f32_tf32     dcn_v2_conv on fp32 tensors with torch's matmul flag off / on: forward, forward + backward
  bf16_off, bf16_on      dcn_v2_conv on a bf16 input with fp32 weight and bias (the autocast case), forward + backward
                         with the flag off / on: the forward is the same, the backward is the FFMA / TF32 one
  ref_tf32               the reference's algorithm with TF32 on (tools/dcn_time.RefAlgo: oracle/_ref/libdcn_ref.so's
                         im2col + torch.matmul), forward and forward + backward; skipped where it was not built
  tv_tf32                torchvision.ops.deform_conv2d with TF32 on, forward and forward + backward (skipped if it does
                         not import)
  split_ieee, split_tf32 the backward's device time per kernel (grad_cols, coord, input, weight, bias, and the rest:
                         the split reduction, the grad_input memset and the up-front copies), from torch.profiler over
                         `reps` calls of dcn.dcn_backward

Each time is tools/devtime.device_ms over `reps` calls after warm-up; the card's name, power limit and max SM clock are
read in the same run.

    python tools/dcn_tf32_time.py [--reps N] [--out PATH]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
import dcn_cases as dc  # noqa: E402
from devtime import card, device_ms  # noqa: E402
from dcn_time import REF_LIB, RefAlgo  # noqa: E402

DEV = "cuda:0"
WARMUP = 2
KERNELS = [("grad_cols", "dcn_grad_cols"), ("coord", "dcn_grad_coord"), ("input", "dcn_grad_input"),
           ("weight", "dcn_grad_weight"), ("bias", "dcn_grad_bias")]


def set_tf32(on):
    torch.backends.cuda.matmul.fp32_precision = "tf32" if on else "ieee"


def backward_split(fn, reps):
    """Device ms per call of each backward kernel of fn, by KERNELS' name prefixes; "other" is everything else."""
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    split = {k: 0.0 for k, _ in KERNELS}
    split["other"] = 0.0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        key = next((k for k, p in KERNELS if p in e.name), "other")
        split[key] += e.device_time / 1000.0 / reps
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dcn_tf32_time.py measures on a CUDA device"
    torch.backends.cudnn.allow_tf32 = False
    ref = RefAlgo() if os.path.exists(REF_LIB) else None
    try:
        import torchvision.ops as tvo
        tvo.deform_conv2d(*(torch.zeros(s, device=DEV) for s in ((1, 1, 3, 3), (1, 18, 3, 3), (1, 1, 3, 3))),
                          padding=1, mask=torch.ones((1, 9, 3, 3), device=DEV))
    except Exception:
        tvo = None
    result = dict(gpu=card(), configs=[])
    for key, B in (("544x736", 1), ("512x512", 1), ("512x512", 16)):
        rows, tot = [], {}
        for layer, c0 in enumerate(dc.DETECTOR[key]):
            c = c0._replace(B=B)
            x, off, m, w, b = (torch.from_numpy(a).to(DEV) for a in dc.make_inputs(c, seed=layer, offsets="random"))
            go = torch.randn((B, c.Co) + dc.out_hw(c), device=DEV)
            st = (c.stride, c.pad, c.dil, c.dg)
            t, split = {}, {}
            for name, on in (("ieee", False), ("tf32", True)):
                set_tf32(on)
                t[f"f32_{name}_fwd"] = device_ms(lambda: pvb.dcn_v2_conv(x, off, m, w, b, *st), args.reps, WARMUP)
                leaves = [v.clone().requires_grad_() for v in (x, off, m, w, b)]
                t[f"f32_{name}_fwd_bwd"] = device_ms(lambda: torch.autograd.grad(pvb.dcn_v2_conv(*leaves, *st), leaves,
                                                                                 go), args.reps, WARMUP)
                xs, offs, ms = (v.bfloat16().requires_grad_() for v in (x, off, m))
                hl = [xs, offs, ms] + [v.clone().requires_grad_() for v in (w, b)]
                gob = go.bfloat16()
                t[f"bf16_{'on' if on else 'off'}_fwd_bwd"] = device_ms(
                    lambda: torch.autograd.grad(pvb.dcn_v2_conv(*hl, *st), hl, gob), args.reps, WARMUP)
                split[name] = {k: round(v, 4) for k, v in backward_split(
                    lambda: pvb.dcn.dcn_backward(x, off, m, w, b, go, *st), args.reps).items()}
            set_tf32(True)
            if ref is not None:
                t["ref_tf32_fwd"] = device_ms(lambda: ref.forward(c, x, off, m, w, b), args.reps, WARMUP)
                t["ref_tf32_fwd_bwd"] = device_ms(lambda: (ref.forward(c, x, off, m, w, b),
                                                           ref.backward(c, x, off, m, w, b, go)), args.reps, WARMUP)
            if tvo is not None:
                tl = [v.clone().requires_grad_() for v in (x, off, m, w, b)]

                def tv_fwd(tl=tl):
                    return tvo.deform_conv2d(tl[0], tl[1], tl[3], tl[4], padding=1, mask=tl[2])
                with torch.no_grad():
                    t["tv_tf32_fwd"] = device_ms(tv_fwd, args.reps, WARMUP)
                t["tv_tf32_fwd_bwd"] = device_ms(lambda: torch.autograd.grad(tv_fwd(), tl, go), args.reps, WARMUP)
            set_tf32(False)
            row = dict(layer=layer, C=c.C, H=c.H, W=c.W, C_out=c.Co, **{k: round(v, 4) for k, v in t.items()},
                       split_ieee=split["ieee"], split_tf32=split["tf32"])
            rows.append(row)
            for k, v in t.items():
                tot[k] = tot.get(k, 0.0) + v
            for name in ("ieee", "tf32"):
                for k, v in split[name].items():
                    tot[f"split_{name}_{k}"] = tot.get(f"split_{name}_{k}", 0.0) + v
            print(json.dumps(dict(config=f"{key} B={B}", **row)), file=sys.stderr, flush=True)
        result["configs"].append(dict(input=key, B=B, layers=rows, sum={k: round(v, 4) for k, v in tot.items()}))
    result["gpu_after"] = card()
    text = json.dumps(result)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)
    print(text)


if __name__ == "__main__":
    main()
