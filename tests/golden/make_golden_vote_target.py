"""Writes tests/golden/vote_target.npz: the fields clean-pvnet's own compute_vertex (lib/utils/pvnet/pvnet_data_utils.py:
30-44) gives for the cases of tests/vote_target_cases.py (K = 1, 9, 17; masks with 0, 1, 2 and 255; keypoints on a pixel,
within 1e-3 of one, at +-1e6 px and at negative coordinates), so the GPU tests do not need the reference checkout.
Case c stores mask{c} uint8 [3,H,W], kpt{c} float64 [3,K,2] and vertex{c} float32 [3,2K,H,W] (the dataset's
`compute_vertex(mask, kpt_2d).transpose(2, 0, 1)` per image).

    PVNET_REFERENCE=/path/to/clean-pvnet python tests/golden/make_golden_vote_target.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from vote_target_cases import case_inputs  # noqa: E402


def reference_compute_vertex(ref_root):
    """compute_vertex from the reference checkout's pvnet_data_utils.py.  The module imports pycocotools and plyfile at
    the top for functions compute_vertex does not use; where they are not installed, empty stand-ins take their place."""
    import importlib
    import importlib.util
    import types
    for name in ("pycocotools", "pycocotools.mask", "plyfile"):
        try:
            importlib.import_module(name)
        except ImportError:
            mod = types.ModuleType(name)
            mod.PlyData = None
            sys.modules[name] = mod
    sys.modules["pycocotools"].mask = sys.modules["pycocotools.mask"]
    path = os.path.join(ref_root, "lib", "utils", "pvnet", "pvnet_data_utils.py")
    spec = importlib.util.spec_from_file_location("reference_pvnet_data_utils", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.compute_vertex


def main():
    compute_vertex = reference_compute_vertex(os.environ.get("PVNET_REFERENCE", "/root/reference"))
    arrays = {}
    for c, (mask, kpt) in enumerate(case_inputs()):
        arrays[f"mask{c}"] = mask
        arrays[f"kpt{c}"] = kpt
        arrays[f"vertex{c}"] = np.stack([compute_vertex(m, k).transpose(2, 0, 1) for m, k in zip(mask, kpt)])
    np.savez_compressed(os.path.join(HERE, "vote_target.npz"), **arrays)


if __name__ == "__main__":
    main()
