#!/usr/bin/env python
"""Times the channels_last half-precision DCNv2 forward (csrc/dcn.cu, DESIGN.md section 8o) at the 16 DCN layers of
the DLA-34 detector, in bf16 and fp16, and prints one JSON object.

Shapes: tests/dcn_cases.DETECTOR at 736x544 (B = 1) and 512x512 (B = 1 and 16), as tools/dcn_half_time.py.  Forward
only, per layer and summed over the 16 layers, in one process on one GPU; every arm's operands are already in the
dtype, so the weight's tap-major copy is the only cast-like work inside a call:

  a_cl        dcn.dcn_forward on channels_last input, offset and mask: the NHWC kernel, channels_last output
  b_nchw      the same call on NCHW copies of the same values: the NCHW kernel
  c_copies    what a channels_last input cost before the NHWC kernel: .contiguous() of input, offset and mask, the
              NCHW kernel, and .contiguous(memory_format=torch.channels_last) of the output
  d_block_cl  a DeformConv block as lib/networks/ct/dla_dcn.py builds it (DCN with its conv_offset_mask, BatchNorm,
              ReLU; eval mode, no autograd) under torch.autocast, the block and its input channels_last
  d_block_nchw the same block and input in NCHW
  ref_f32     the reference's algorithm, fp32 (tools/dcn_time.RefAlgo: oracle/_ref/libdcn_ref.so's im2col + fp32
              torch.matmul, TF32 off)
  ref_bf16    the same im2col, its columns cast to bf16, then a bf16 torch.matmul + the bias ("im2col + cuBLAS")

The ref arms do not depend on the dtype and are timed once per layer; they are skipped where the library was not
built.  Arms a, b and c are timed twice, alternating, and each keeps its faster reading.  Each time is
tools/devtime.device_ms over `reps` calls after warm-up; the card's name, power limit and max SM clock are read in
the same run.

    python tools/dcn_nhwc_time.py [--reps N] [--out PATH]
"""
import argparse
import copy
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
from torch import nn  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
import dcn_cases as dc  # noqa: E402
from devtime import card, device_ms  # noqa: E402
from dcn_time import REF_LIB, RefAlgo  # noqa: E402

DEV = "cuda:0"
WARMUP = 2
CL = torch.channels_last
DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}


def block(c):
    """DCN 3x3 -> BatchNorm -> ReLU (dla_dcn.py's DeformConv) with a non-zero offset branch, eval mode."""
    torch.manual_seed(0)
    net = nn.Sequential(pvb.DCN(c.C, c.Co, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1),
                        nn.BatchNorm2d(c.Co), nn.ReLU(inplace=True)).to(DEV).eval()
    with torch.no_grad():
        net[0].conv_offset_mask.weight.normal_(0, 0.01)
        net[0].conv_offset_mask.bias.normal_(0, 0.5)
    return net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dcn_nhwc_time.py measures on a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ref = RefAlgo() if os.path.exists(REF_LIB) else None
    fwd = pvb.dcn.dcn_forward

    def ms(fn):
        return device_ms(fn, args.reps, WARMUP)

    result = dict(gpu=card(), configs=[])
    for key, B in (("544x736", 1), ("512x512", 1), ("512x512", 16)):
        rows, tot = [], {}
        for layer, c0 in enumerate(dc.DETECTOR[key]):
            c = c0._replace(B=B)
            x, off, m, w, b = (torch.from_numpy(a).to(DEV) for a in dc.make_inputs(c, seed=layer, offsets="random"))
            st = (c.stride, c.pad, c.dil, c.dg)
            t = {}
            net = block(c)
            net_cl = copy.deepcopy(net).to(memory_format=CL)
            for name, dt in DTYPES.items():
                xs, offs, ms_, ws, bs = (v.to(dt) for v in (x, off, m, w, b))
                xc, offc, mc = (v.contiguous(memory_format=CL) for v in (xs, offs, ms_))
                arms = {
                    "a_cl": lambda: fwd(xc, offc, mc, ws, bs, *st),
                    "b_nchw": lambda: fwd(xs, offs, ms_, ws, bs, *st),
                    "c_copies": lambda: fwd(xc.contiguous(), offc.contiguous(), mc.contiguous(), ws, bs,
                                            *st).contiguous(memory_format=CL),
                }
                assert fwd(xc, offc, mc, ws, bs, *st).is_contiguous(memory_format=CL)
                for arm in arms:
                    t[f"{arm}_{name}"] = float("inf")
                for _ in range(2):
                    for arm, fn in arms.items():
                        t[f"{arm}_{name}"] = min(t[f"{arm}_{name}"], ms(fn))

                def run_block(n, inp, dt=dt):
                    with torch.no_grad(), torch.autocast("cuda", dtype=dt):
                        return n(inp)
                t[f"d_block_cl_{name}"] = ms(lambda: run_block(net_cl, xc))
                t[f"d_block_nchw_{name}"] = ms(lambda: run_block(net, xs))
            if ref is not None:
                t["ref_f32"] = ms(lambda: ref.forward(c, x, off, m, w, b))
                wl, bl = w.reshape(c.Co, -1).bfloat16(), b.bfloat16()
                Ho, Wo = dc.out_hw(c)

                def ref_bf16():
                    cols = torch.empty((B, c.C * c.kh * c.kw, Ho * Wo), device=DEV)
                    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
                    ref.lib.modulated_deformable_im2col_cuda(s, ref._p(x), ref._p(off), ref._p(m), *ref._g(c, B),
                                                             ref._p(cols))
                    return bl[None, :, None] + torch.matmul(wl, cols.bfloat16())
                t["ref_bf16"] = ms(ref_bf16)
            row = dict(layer=layer, C=c.C, H=c.H, W=c.W, C_out=c.Co, **{k: round(v, 4) for k, v in t.items()})
            rows.append(row)
            for k, v in t.items():
                tot[k] = tot.get(k, 0.0) + v
            print(json.dumps(dict(config=f"{key} B={B}", **row)), file=sys.stderr, flush=True)
        tot = {k: round(v, 4) for k, v in tot.items()}
        for name in DTYPES:
            tot[f"a_over_c_{name}"] = round(tot[f"a_cl_{name}"] / tot[f"c_copies_{name}"], 4)
            tot[f"a_over_b_{name}"] = round(tot[f"a_cl_{name}"] / tot[f"b_nchw_{name}"], 4)
        result["configs"].append(dict(input=key, B=B, layers=rows, sum=tot))
    result["gpu_after"] = card()
    text = json.dumps(result)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)
    print(text)


if __name__ == "__main__":
    main()
