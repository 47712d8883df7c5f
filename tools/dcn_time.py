#!/usr/bin/env python
"""Times the DCNv2 kernels (csrc/dcn.cu) at the 16 DCN layers of the DLA-34 detector and prints one JSON object.

Shapes: tests/dcn_cases.DETECTOR at 736x544 (B = 1) and 512x512 (B = 1 and 16); forward alone, and forward + backward
(all five gradients).  Per shape and summed over the 16 layers (one detector pass), in the same process on the same GPU:

  ours         pvb.dcn.dcn_forward / dcn_backward
  reference    the reference's algorithm rebuilt from oracle/_ref/libdcn_ref.so (oracle/build_dcn_ref.py): its im2col
               launcher for the whole batch + fp32 torch.matmul with TF32 off + the bias (dcn_v2_cuda.cu:43); backward
               per image as dcn_v2_cuda.cu:259-330 loops: W^T grad_out, col2im_coord, col2im, im2col, grad_out cols^T,
               the bias sum (skipped where the library was not built)
  torchvision  torchvision.ops.deform_conv2d (skipped if it does not import)

CUDA events around `reps` calls after warm-up.  The FP32 rate counts 2*C_out*C*kh*kw*Ho*Wo*B FLOP for the forward and
three times that for forward + backward (grad_cols and grad_weight are GEMMs of the same size), against the H100 SXM
data sheet's 67 TFLOP/s FP32; the card name, power limit and max SM clock are read in the same call.

    python tools/dcn_time.py [--reps N] [--out PATH]
"""
import argparse
import ctypes
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

REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libdcn_ref.so")
PEAK_FP32 = 67e12
DEV = "cuda:0"
WARMUP = 2


class RefAlgo:
    """The reference's forward and backward on its own launchers + fp32 matmul (TF32 off)."""

    def __init__(self):
        lib = ctypes.CDLL(REF_LIB)
        i, p = ctypes.c_int, ctypes.c_void_p
        lib.modulated_deformable_im2col_cuda.argtypes = [p, p, p, p] + [i] * 15 + [p]
        lib.modulated_deformable_col2im_cuda.argtypes = [p, p, p, p] + [i] * 15 + [p]
        lib.modulated_deformable_col2im_coord_cuda.argtypes = [p, p, p, p, p] + [i] * 15 + [p, p]
        self.lib = lib

    @staticmethod
    def _g(c, B):
        Ho, Wo = dc.out_hw(c)
        return [B, c.C, c.H, c.W, Ho, Wo, c.kh, c.kw, c.pad[0], c.pad[1], c.stride[0], c.stride[1], c.dil[0], c.dil[1],
                c.dg]

    @staticmethod
    def _p(t):
        return ctypes.c_void_p(t.data_ptr())

    def forward(self, c, x, off, m, w, b):
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        Ho, Wo = dc.out_hw(c)
        cols = torch.empty((c.B, c.C * c.kh * c.kw, Ho * Wo), device=DEV)
        self.lib.modulated_deformable_im2col_cuda(s, self._p(x), self._p(off), self._p(m), *self._g(c, c.B), self._p(cols))
        return (b[None, :, None] + torch.matmul(w.reshape(c.Co, -1), cols)).reshape(c.B, c.Co, Ho, Wo)

    def backward(self, c, x, off, m, w, b, go):
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        Ho, Wo = dc.out_hw(c)
        W2 = w.reshape(c.Co, -1)
        gi, goff, gm = torch.zeros_like(x), torch.zeros_like(off), torch.zeros_like(m)
        gw, gb = torch.zeros_like(W2), torch.zeros_like(b)
        cols = torch.empty((c.C * c.kh * c.kw, Ho * Wo), device=DEV)
        g1 = self._g(c, 1)
        for i in range(c.B):
            gon = go[i].reshape(c.Co, -1)
            torch.matmul(W2.t(), gon, out=cols)
            self.lib.modulated_deformable_col2im_coord_cuda(s, self._p(cols), self._p(x[i]), self._p(off[i]),
                                                            self._p(m[i]), *g1, self._p(goff[i]), self._p(gm[i]))
            self.lib.modulated_deformable_col2im_cuda(s, self._p(cols), self._p(off[i]), self._p(m[i]), *g1,
                                                      self._p(gi[i]))
            self.lib.modulated_deformable_im2col_cuda(s, self._p(x[i]), self._p(off[i]), self._p(m[i]), *g1,
                                                      self._p(cols))
            gw.addmm_(gon, cols.t())
            gb.add_(gon.sum(1))
        return gi, goff, gm, gw, gb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dcn_time.py measures on a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ref = RefAlgo() if os.path.exists(REF_LIB) else None
    try:
        import torchvision.ops as tvo
        tvo.deform_conv2d(*(torch.zeros(s, device=DEV) for s in ((1, 1, 3, 3), (1, 18, 3, 3), (1, 1, 3, 3))),
                          padding=1, mask=torch.ones((1, 9, 3, 3), device=DEV))
    except Exception:
        tvo = None
    result = dict(gpu=card(), peak_fp32_tflops=PEAK_FP32 / 1e12, configs=[])
    for key, B in (("544x736", 1), ("512x512", 1), ("512x512", 16)):
        rows, tot = [], {}
        for layer, c0 in enumerate(dc.DETECTOR[key]):
            c = c0._replace(B=B)
            x, off, m, w, b = (torch.from_numpy(a).to(DEV) for a in dc.make_inputs(c, seed=layer, offsets="random"))
            go = torch.randn((B, c.Co) + dc.out_hw(c), device=DEV)
            flop = 2.0 * c.Co * c.C * c.kh * c.kw * c.H * c.W * B
            st = (c.stride, c.pad, c.dil, c.dg)
            t = dict(ours_fwd=device_ms(lambda: pvb.dcn.dcn_forward(x, off, m, w, b, *st), args.reps, WARMUP),
                     ours_fwd_bwd=device_ms(lambda: (pvb.dcn.dcn_forward(x, off, m, w, b, *st),
                                                     pvb.dcn.dcn_backward(x, off, m, w, b, go, *st)), args.reps, WARMUP))
            if ref is not None:
                t["ref_fwd"] = device_ms(lambda: ref.forward(c, x, off, m, w, b), args.reps, WARMUP)
                t["ref_fwd_bwd"] = device_ms(lambda: (ref.forward(c, x, off, m, w, b),
                                                      ref.backward(c, x, off, m, w, b, go)), args.reps, WARMUP)
            if tvo is not None:
                xs, offs, ms, ws, bs = (v.clone().requires_grad_() for v in (x, off, m, w, b))
                t["tv_fwd"] = device_ms(lambda: tvo.deform_conv2d(x, off, w, b, padding=1, mask=m), args.reps, WARMUP)
                t["tv_fwd_bwd"] = device_ms(lambda: torch.autograd.grad(
                    tvo.deform_conv2d(xs, offs, ws, bs, padding=1, mask=ms), (xs, offs, ms, ws, bs), go),
                    args.reps, WARMUP)
            row = dict(layer=layer, C=c.C, H=c.H, W=c.W, C_out=c.Co, gflop_fwd=flop / 1e9,
                       **{k: round(v, 4) for k, v in t.items()},
                       ours_fwd_tflops=round(flop / t["ours_fwd"] / 1e9, 2),
                       ours_fwd_bwd_tflops=round(3 * flop / t["ours_fwd_bwd"] / 1e9, 2))
            rows.append(row)
            for k, v in t.items():
                tot[k] = tot.get(k, 0.0) + v
            tot["gflop_fwd"] = tot.get("gflop_fwd", 0.0) + flop / 1e9
            print(json.dumps(dict(config=f"{key} B={B}", **row)), file=sys.stderr, flush=True)
        tot = {k: round(v, 4) for k, v in tot.items()}
        tot["ours_fwd_share_of_peak"] = round(tot["gflop_fwd"] * 1e9 / (tot["ours_fwd"] * 1e-3) / PEAK_FP32, 4)
        tot["ours_fwd_bwd_share_of_peak"] = round(3 * tot["gflop_fwd"] * 1e9 / (tot["ours_fwd_bwd"] * 1e-3) / PEAK_FP32, 4)
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
