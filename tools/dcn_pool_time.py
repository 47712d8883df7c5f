#!/usr/bin/env python
"""Times DCNv2's deformable PSROI pooling (csrc/dcn_pool.cu) against the reference's own kernels and prints one JSON
line.

Shapes: a detector head (B = 2, C = 256, 50x68 map, 2x512 ROIs, P = 7, scale 1/16, sample_per_part 2 and 4) and
lib/csrc/dcn_v2/test.py's example_dpooling ([2,32,64,64], 20 ROIs, P = 7, scale 1/4), each with and without offsets;
forward alone, and forward + backward.  In the same process on the same GPU:

  ours        pvb.dcn_pool.pool_forward / pool_backward (the backward recomputes the counts)
  reference   oracle/_ref/libdcn_pool_ref.so (oracle/build_dcn_pool_ref.py), launched as its host functions launch it,
              with the output, count and gradients zeroed first as they are (skipped where the library was not built)

Times come from tools/devtime.device_ms (CUDA events around `reps` calls after warm-up); the card name, power limit and
max SM clock are read in the same run.

    python tools/dcn_pool_time.py [--reps N] [--out PATH]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import clean_pvnet_b200 as pvb  # noqa: E402
from devtime import card, device_ms  # noqa: E402

REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libdcn_pool_ref.so")
DEV = "cuda:0"
WARMUP = 3


def inputs(seed, B, C, H, W, n, span, size):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g)
    xy = torch.randint(span, (n, 2), generator=g).float()
    wh = torch.randint(size, (n, 2), generator=g).float()
    rois = torch.cat((torch.randint(B, (n, 1), generator=g).float(), xy, xy + wh), 1)
    trans = torch.randn(n, 2, 7, 7, generator=g)
    return x.to(DEV), rois.to(DEV), trans.to(DEV)


class Ref:
    def __init__(self):
        lib = ctypes.CDLL(REF_LIB)
        i, p, f = ctypes.c_int, ctypes.c_void_p, ctypes.c_float
        lib.ref_dcn_pool_forward.argtypes = [p] * 5 + [i] * 9 + [f, f, p]
        lib.ref_dcn_pool_backward.argtypes = [p] * 7 + [i] * 9 + [f, f, p]
        self.lib = lib

    @staticmethod
    def _p(t):
        return ctypes.c_void_p(t.data_ptr())

    def forward(self, x, rois, trans, no_trans, k):
        n, (B, C, H, W), P = rois.shape[0], x.shape, k["pooled_size"]
        out = torch.zeros((n, C, P, P), device=DEV)
        cnt = torch.zeros_like(out)
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.lib.ref_dcn_pool_forward(self._p(x), self._p(rois), self._p(trans), self._p(out), self._p(cnt), n, C, H, W,
                                      P, P, k["sample_per_part"], 1, int(no_trans), k["spatial_scale"], k["trans_std"], s)
        return out, cnt

    def backward(self, go, cnt, x, rois, trans, no_trans, k):
        n, (B, C, H, W), P = rois.shape[0], x.shape, k["pooled_size"]
        gi, gt = torch.zeros_like(x), torch.zeros_like(trans)
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.lib.ref_dcn_pool_backward(self._p(go), self._p(cnt), self._p(x), self._p(rois), self._p(trans), self._p(gi),
                                       self._p(gt), n, C, H, W, P, P, k["sample_per_part"], 1, int(no_trans),
                                       k["spatial_scale"], k["trans_std"], s)
        return gi, gt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dcn_pool_time.py measures on a CUDA device"
    ref = Ref() if os.path.exists(REF_LIB) else None
    shapes = [("detector_head_spp2", (5, 2, 256, 50, 68, 1024, 900, 400), 1 / 16, 2),
              ("detector_head_spp4", (5, 2, 256, 50, 68, 1024, 900, 400), 1 / 16, 4),
              ("example_dpooling", (1, 2, 32, 64, 64, 20, 256, 64), 1 / 4, 4)]
    result = dict(gpu=card(), reps=args.reps, configs=[])
    for name, shp, scale, spp in shapes:
        x, rois, trans = inputs(*shp)
        k = dict(spatial_scale=scale, pooled_size=7, output_dim=shp[2], group_size=1, part_size=7,
                 sample_per_part=spp, trans_std=0.1)
        for no_trans in (True, False):
            go = torch.randn((shp[5], shp[2], 7, 7), device=DEV)

            def ours_f():
                return pvb.dcn_pool.pool_forward(x, rois, trans, no_trans=no_trans, **k)

            def ours_fb():
                ours_f()
                return pvb.dcn_pool.pool_backward(go, x, rois, trans, no_trans=no_trans, **k)

            t = dict(ours_fwd_ms=device_ms(ours_f, args.reps, WARMUP), ours_fwd_bwd_ms=device_ms(ours_fb, args.reps,
                                                                                                  WARMUP))
            if ref is not None:
                def ref_f():
                    return ref.forward(x, rois, trans, no_trans, k)

                def ref_fb():
                    _, cnt = ref_f()
                    return ref.backward(go, cnt, x, rois, trans, no_trans, k)

                t["ref_fwd_ms"] = device_ms(ref_f, args.reps, WARMUP)
                t["ref_fwd_bwd_ms"] = device_ms(ref_fb, args.reps, WARMUP)
                t["fwd_speedup"] = t["ref_fwd_ms"] / t["ours_fwd_ms"]
                t["fwd_bwd_speedup"] = t["ref_fwd_bwd_ms"] / t["ours_fwd_bwd_ms"]
            result["configs"].append(dict(config=name, no_trans=no_trans, B=shp[1], C=shp[2], H=shp[3], W=shp[4],
                                          n_roi=shp[5], sample_per_part=spp, spatial_scale=scale,
                                          **{key: round(v, 4) for key, v in t.items()}))
    text = json.dumps(result)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)
    print(text)


if __name__ == "__main__":
    main()
