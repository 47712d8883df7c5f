"""Writes tests/golden/ct_decode.npz: what clean-pvnet's own Network.decode_detection computes
(lib/networks/ct/dla.py:20-26: torch.sigmoid, lib/utils/ct/ct_decode.py decode_ct_hm, data_utils.clip_to_image) for the
tie-free cases of tests/ct_decode_cases.py, on CPU torch, and the image-frame boxes its consumers derive from them with
data_utils.get_affine_transform / affine_transform.  Only tie-free cases are stored: CPU torch's topk orders equal values
differently from CUDA torch's.  Case c stores logits{c} float32 [B,C,H,W], wh{c} float32 [B,2,H,W], K{c}, ct{c} float32
[B,K,2], detection{c} float32 [B,K,6] and boxes{c} float64 [B,K,4] (for input size BOX_INPUT_SIZE, centre BOX_CENTER and
scale BOX_SCALE), plus names.

    PVNET_REFERENCE=/path/to/clean-pvnet python tests/golden/make_golden_ct_decode.py
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from ct_decode_cases import BOX_CENTER, BOX_INPUT_SIZE, BOX_SCALE, golden_cases  # noqa: E402
from make_golden_ct_target import reference_data_utils  # noqa: E402


def reference_modules(ref_root):
    """(data_utils, ct_decode) from the reference checkout; ct_decode imports data_utils as lib.utils.data_utils."""
    import types
    du = reference_data_utils(ref_root)
    for name in ("lib", "lib.utils"):
        if name not in sys.modules:
            mod = types.ModuleType(name)
            mod.__path__ = []
            sys.modules[name] = mod
    sys.modules["lib.utils"].data_utils = du
    sys.modules["lib.utils.data_utils"] = du
    spec = importlib.util.spec_from_file_location("reference_ct_decode", os.path.join(ref_root, "lib", "utils", "ct",
                                                                                      "ct_decode.py"))
    cd = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cd)
    return du, cd


def main():
    ref = os.environ.get("PVNET_REFERENCE")
    if not ref:
        sys.exit("set PVNET_REFERENCE to a clean-pvnet checkout")
    du, cd = reference_modules(ref)
    out = {}
    names = []
    w, h = BOX_INPUT_SIZE
    trans = du.get_affine_transform(np.array(BOX_CENTER, np.float32), np.array(BOX_SCALE, np.float64), 0, [w, h], inv=1)
    for c, (name, lg, wh, K) in enumerate(golden_cases()):
        hm = torch.from_numpy(lg)
        ct, det = cd.decode_ct_hm(torch.sigmoid(hm), torch.from_numpy(wh), K=K)
        det[..., :4] = du.clip_to_image(det[..., :4], hm.shape[2], hm.shape[3])
        box = det[..., :4].numpy() * 4
        boxes = np.stack([np.stack([du.affine_transform(bx.reshape(-1, 2), trans).ravel() for bx in img]) for img in box])
        out.update({f"logits{c}": lg, f"wh{c}": wh, f"K{c}": np.int64(K), f"ct{c}": ct.numpy(),
                    f"detection{c}": det.numpy(), f"boxes{c}": boxes.astype(np.float64)})
        names.append(name)
    out["names"] = np.array(names)
    path = os.path.join(HERE, "ct_decode.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
