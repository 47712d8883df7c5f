"""Writes tests/golden/ct_target.npz: the heatmaps clean-pvnet's own data_utils.gaussian_radius and draw_umich_gaussian
(lib/utils/data_utils.py:10-64) give for the cases of tests/ct_target_cases.py, drawn the way the CenterNet datasets'
prepare_detection draws them (lib/datasets/tless/ct.py:72-92), so the GPU tests do not need the reference checkout.
Case c stores ct_ind{c} int64 [B,M], ct_radius{c} int32 [B,M], ct_cls{c} int64 [B,M], ct_01{c} float32 [B,M],
wh{c} float64 [B,M,2] and ct_hm{c} float32 [B,C,H,W].  It also stores radius_table int32 [256,256], the radius of every
integer (h, w) in [1, 256]^2 at [h - 1, w - 1], and edge_wh float64 [n,2] / edge_radius int32 [n], float sizes just
above, at and below integers.

    PVNET_REFERENCE=/path/to/clean-pvnet python tests/golden/make_golden_ct_target.py
"""
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from ct_target_cases import case_images, pack  # noqa: E402

EDGE_SIZES = [1.0, 1.0 + 1e-9, 7.0000001, 7.0, 6.9999999, 12.5, 0.3, 0.0, 31.0000002, 100.00001, 255.99999, 2.0 ** -30]


def reference_data_utils(ref_root):
    """lib/utils/data_utils.py from the reference checkout.  It imports imgaug and lib.config at the top for functions
    the heatmap does not use; empty stand-ins take their place where they are not importable."""
    import importlib
    import importlib.util
    import types
    try:
        importlib.import_module("imgaug")
    except ImportError:
        ia = types.ModuleType("imgaug")
        ia.augmenters = types.ModuleType("imgaug.augmenters")
        sys.modules["imgaug"], sys.modules["imgaug.augmenters"] = ia, ia.augmenters
    if "lib.config" not in sys.modules:
        for name in ("lib", "lib.config"):
            mod = types.ModuleType(name)
            mod.__path__ = []
            sys.modules[name] = mod
        sys.modules["lib.config"].cfg = types.SimpleNamespace()
    path = os.path.join(ref_root, "lib", "utils", "data_utils.py")
    spec = importlib.util.spec_from_file_location("reference_data_utils", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_radius(du):
    """prepare_detection's radius rule with the reference's gaussian_radius, on float64 h and w."""
    return lambda h, w: max(0, int(du.gaussian_radius((math.ceil(h), math.ceil(w)))))


def reference_ct_hm(du, ind, rad, cls, c01, C, H, W):
    """The dataset's ct_hm per image: draw_umich_gaussian(ct_hm[cls], (cx, cy), r) per object, in object order."""
    out = np.zeros((ind.shape[0], C, H, W), np.float32)
    for b in range(ind.shape[0]):
        for j in range(ind.shape[1]):
            if c01[b, j] == 1:
                cy, cx = divmod(int(ind[b, j]), W)
                du.draw_umich_gaussian(out[b, int(cls[b, j])], np.array([cx, cy], np.int32), int(rad[b, j]))
    return out


def main():
    du = reference_data_utils(os.environ.get("PVNET_REFERENCE", "/root/reference"))
    radius = reference_radius(du)
    arrays = {}
    for c, (B, C, H, W, images) in enumerate(case_images()):
        ind, rad, cls, c01, wh = pack(images, W, radius)
        arrays.update({f"ct_ind{c}": ind, f"ct_radius{c}": rad, f"ct_cls{c}": cls, f"ct_01{c}": c01, f"wh{c}": wh,
                       f"ct_hm{c}": reference_ct_hm(du, ind, rad, cls, c01, C, H, W)})
    arrays["radius_table"] = np.array([[radius(h, w) for w in range(1, 257)] for h in range(1, 257)], np.int32)
    edge = np.array([(w, h) for h in EDGE_SIZES for w in EDGE_SIZES], np.float64)
    arrays["edge_wh"] = edge
    arrays["edge_radius"] = np.array([radius(h, w) for w, h in edge], np.int32)
    np.savez_compressed(os.path.join(HERE, "ct_target.npz"), **arrays)


if __name__ == "__main__":
    main()
