#!/usr/bin/env python
"""Times the half-precision DCNv2 forward (csrc/dcn.cu, DESIGN.md section 8n) at the 16 DCN layers of the DLA-34
detector and prints one JSON object.

Shapes: tests/dcn_cases.DETECTOR at 736x544 (B = 1) and 512x512 (B = 1 and 16), as tools/dcn_time.py.  Forward alone
and forward + backward (all five gradients), per layer and summed over the 16 layers, in one process on one GPU:

  ours_bf16, ours_f16  dcn_v2_conv on a bf16 / fp16 input with fp32 weight and bias (the autocast case: the casts and
                       the weight's tap-major copy are inside the timed call); its backward is the fp32 one on up-casts
  ours_bf16_call, ...  dcn.dcn_forward on operands already in the dtype (no autograd, no casts; the weight's
                       tap-major copy is still inside): the cost of the call itself
  ours_f32             dcn_v2_conv on fp32 tensors (the FP32-FFMA kernels)
  ref_f32              the reference's algorithm (tools/dcn_time.RefAlgo: oracle/_ref/libdcn_ref.so's im2col + fp32
                       torch.matmul, TF32 off; its per-image backward)
  ref_bf16             the same im2col, its columns cast to bf16, then a bf16 torch.matmul + the bias: the
                       "im2col + cuBLAS" rival of the new path (forward only)
  tv_autocast          torchvision.ops.deform_conv2d under torch.autocast("cuda", bfloat16) (skipped if it does not
                       import)

The ref arms are skipped where the library was not built.  Each time is tools/devtime.device_ms over `reps` calls after
warm-up.  The forward's share of peak counts 2*C_out*C*kh*kw*Ho*Wo*B FLOP against the H100 SXM data sheet's 989 TFLOP/s
dense BF16 / FP16; the card's name, power limit and max SM clock are read in the same run.

    python tools/dcn_half_time.py [--reps N] [--out PATH]
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

PEAK_HALF = 989e12
DEV = "cuda:0"
WARMUP = 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dcn_half_time.py measures on a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ref = RefAlgo() if os.path.exists(REF_LIB) else None
    try:
        import torchvision.ops as tvo
        tvo.deform_conv2d(*(torch.zeros(s, device=DEV) for s in ((1, 1, 3, 3), (1, 18, 3, 3), (1, 1, 3, 3))),
                          padding=1, mask=torch.ones((1, 9, 3, 3), device=DEV))
    except Exception:
        tvo = None
    result = dict(gpu=card(), peak_half_tflops=PEAK_HALF / 1e12, configs=[])
    for key, B in (("544x736", 1), ("512x512", 1), ("512x512", 16)):
        rows, tot = [], {}
        for layer, c0 in enumerate(dc.DETECTOR[key]):
            c = c0._replace(B=B)
            x, off, m, w, b = (torch.from_numpy(a).to(DEV) for a in dc.make_inputs(c, seed=layer, offsets="random"))
            go = torch.randn((B, c.Co) + dc.out_hw(c), device=DEV)
            flop = 2.0 * c.Co * c.C * c.kh * c.kw * c.H * c.W * B
            st = (c.stride, c.pad, c.dil, c.dg)
            t = {}
            for name, dt in (("ours_bf16", torch.bfloat16), ("ours_f16", torch.float16), ("ours_f32", torch.float32)):
                xs, offs, ms = (v.to(dt) for v in (x, off, m))
                gos = go.to(dt)
                t[name + "_fwd"] = device_ms(lambda: pvb.dcn_v2_conv(xs, offs, ms, w, b, *st), args.reps, WARMUP)
                if dt != torch.float32:      # the same forward on operands already in the dtype, without autograd
                    wl, bl = w.to(dt), b.to(dt)
                    t[name + "_call_fwd"] = device_ms(lambda: pvb.dcn.dcn_forward(xs, offs, ms, wl, bl, *st),
                                                      args.reps, WARMUP)
                leaves = [v.clone().requires_grad_() for v in (xs, offs, ms, w, b)]
                t[name + "_fwd_bwd"] = device_ms(lambda: torch.autograd.grad(pvb.dcn_v2_conv(*leaves, *st), leaves, gos),
                                                 args.reps, WARMUP)
            if ref is not None:
                t["ref_f32_fwd"] = device_ms(lambda: ref.forward(c, x, off, m, w, b), args.reps, WARMUP)
                t["ref_f32_fwd_bwd"] = device_ms(lambda: (ref.forward(c, x, off, m, w, b),
                                                          ref.backward(c, x, off, m, w, b, go)), args.reps, WARMUP)
                wl, bl = w.reshape(c.Co, -1).bfloat16(), b.bfloat16()
                Ho, Wo = dc.out_hw(c)

                def ref_bf16():
                    cols = torch.empty((B, c.C * c.kh * c.kw, Ho * Wo), device=DEV)
                    ref.lib.modulated_deformable_im2col_cuda(ref_stream(), ref._p(x), ref._p(off), ref._p(m),
                                                             *ref._g(c, B), ref._p(cols))
                    return bl[None, :, None] + torch.matmul(wl, cols.bfloat16())
                t["ref_bf16_fwd"] = device_ms(ref_bf16, args.reps, WARMUP)
            if tvo is not None:
                xs, offs, ms, ws, bs = (v.clone().requires_grad_() for v in (x, off, m, w, b))

                def tv_fwd(xs=xs, offs=offs, ms=ms, ws=ws, bs=bs):
                    with torch.autocast("cuda", dtype=torch.bfloat16):
                        return tvo.deform_conv2d(xs, offs, ws, bs, padding=1, mask=ms)
                with torch.no_grad():
                    t["tv_autocast_fwd"] = device_ms(tv_fwd, args.reps, WARMUP)
                t["tv_autocast_fwd_bwd"] = device_ms(lambda: torch.autograd.grad(tv_fwd(), (xs, offs, ms, ws, bs), go),
                                                     args.reps, WARMUP)
            row = dict(layer=layer, C=c.C, H=c.H, W=c.W, C_out=c.Co, gflop_fwd=flop / 1e9,
                       **{k: round(v, 4) for k, v in t.items()},
                       ours_bf16_fwd_tflops=round(flop / t["ours_bf16_fwd"] / 1e9, 2))
            rows.append(row)
            for k, v in t.items():
                tot[k] = tot.get(k, 0.0) + v
            tot["gflop_fwd"] = tot.get("gflop_fwd", 0.0) + flop / 1e9
            print(json.dumps(dict(config=f"{key} B={B}", **row)), file=sys.stderr, flush=True)
        tot = {k: round(v, 4) for k, v in tot.items()}
        for name in ("ours_bf16", "ours_f16"):
            tot[name + "_fwd_share_of_peak"] = round(tot["gflop_fwd"] * 1e9 / (tot[name + "_fwd"] * 1e-3) / PEAK_HALF, 4)
        result["configs"].append(dict(input=key, B=B, layers=rows, sum=tot))
    result["gpu_after"] = card()
    text = json.dumps(result)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)
    print(text)


def ref_stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


if __name__ == "__main__":
    main()
