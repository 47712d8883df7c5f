#!/usr/bin/env python
"""Hashes (SHA-256) the pruned v3 vote's workspace regions after bench.py-shaped calls (hn = 512, t = 0.99), so two
builds of the prune kernels can be compared byte for byte: prune_key, both pass lists within their lengths, prune_len, the cell
records, the sub-cell records (an empty sub-cell's last word alone, which is all that is written of it) and the
sub-cell bounds B2 (zero except for pass-2 candidates).  The sub-cell regions sit at the offsets
tests/test_gpu_prune_subcell.py reads them from.  One call per seed: inputs from synth.make_inputs(workload, seed),
vote seed 1000 + the seed's position.

    python tools/prune_regions_dump.py --workload cfg2|cfg4 [--seeds 1236 1237 1238] --out FILE.json
    python tools/prune_regions_dump.py --compare A.json B.json
"""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

HN, THRESH = 512, 0.99


def dump(workload, seeds, out):
    import torch
    import clean_pvnet_b200 as pvb
    from clean_pvnet_b200 import _lib, synth, ransac_voting_gpu as rv
    if not torch.cuda.is_available():
        raise SystemExit("prune_regions_dump.py needs a CUDA device")
    lib = _lib.load()
    res = {}
    for i, s in enumerate(seeds):
        mask, vertex, _ = synth.make_inputs(workload, device="cuda:0", seed=s)
        pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=THRESH, seed=1000 + i)
        torch.cuda.synchronize()
        m, v = rv._check_inputs(mask, vertex)
        d = rv._make_desc(m, v, HN, THRESH, 5, 30000, _lib.PVB_SELECT_BYTE, 1000 + i, 0, None)
        ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
        L = _lib.PvbLayout()
        _lib.check(lib.pvb_workspace_layout(d, L))
        B, K, nc = d.B, d.K, L.prune_ncells
        rec = 4 + 128 // 2

        def ints(off, n):
            return ws[off:off + 4 * n].view(torch.int32).cpu().numpy()
        sub_off = (L.prune_len + 2 * B * K * 4 + 255) // 256 * 256
        nsub = B * K * nc * 4 * rec
        b2_off = (sub_off + 4 * nsub + 255) // 256 * 256
        lens = ints(L.prune_len, 2 * B * K).reshape(2, B, K)
        lists = ints(L.prune_list, 2 * B * K * HN).reshape(2, B, K, HN).copy()
        lists[np.arange(HN) >= lens[..., None]] = -1
        sub = ints(sub_off, nsub).reshape(B, K, nc, 4, rec).copy()
        sub[..., :-1][(sub[..., -1] >> 16) == 0] = 0
        regions = dict(key=ints(L.prune_key, B * K * HN), lists=lists, len=lens,
                       cells=ints(L.prune_cells, B * K * nc * rec), sub=sub, b2=ints(b2_off, B * K * HN))
        for name, arr in regions.items():
            res[f"{workload}/{s}/{name}"] = [hashlib.sha256(np.ascontiguousarray(arr).tobytes()).hexdigest(), arr.nbytes]
        print(f"{workload} seed {s}: pass lengths {lens[0].mean():.1f} + {lens[1].mean():.1f} per (image, keypoint)")
    with open(out, "w") as fh:
        json.dump(res, fh, indent=1)


def compare(a, b):
    x, y = (json.load(open(f)) for f in (a, b))
    if sorted(x) != sorted(y):
        raise SystemExit(f"different regions: {sorted(x)} vs {sorted(y)}")
    bad = [k for k in sorted(x) if x[k] != y[k]]
    for k in sorted(x):
        print(f"{k:>22}: {'byte-equal' if k not in bad else 'DIFFERENT'} ({x[k][1]} bytes)")
    return not bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=["cfg2", "cfg4"])
    ap.add_argument("--seeds", type=int, nargs="+", default=[1236, 1237, 1238])
    ap.add_argument("--out", default=None, help="JSON file of the region hashes")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    if not args.out:
        raise SystemExit("--out FILE.json is required")
    dump(args.workload, args.seeds, args.out)


if __name__ == "__main__":
    main()
