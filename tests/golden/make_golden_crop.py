"""Writes tests/golden/tless_crop.npz: the outputs of clean-pvnet's own T-LESS crop and un-crop code on seeded 720x540
images -- tless_test_utils.pvnet_transform (lib/utils/tless/tless_test_utils.py:57-77) for each box, and
data_utils.affine_transform(kpt, data_utils.get_affine_transform(center, scale, 0, [w, h], inv=1)) as the evaluator
maps keypoints back (lib/evaluators/tless_test/pvnet.py:229-239) -- at both T-LESS configurations (input 256, scale
ratio 2.4, box ratio 1.2; input 128, 1.2, 1.1), including degenerate (zero-size) boxes.

    PVNET_REFERENCE=/path/to/clean-pvnet python tests/golden/make_golden_crop.py

`lib.config` is replaced by a stub that holds only cfg.tless (its real module parses the command line), and `imgaug`,
which only the training augmentation uses, by inert constructors.  The images are integer patterns rebuilt from their
stored parameters (crop_cases.pattern_images), and the float32 inputs are stored as a SHA-256 digest per box (bit-exact,
64 bytes instead of 0.8 MB), so the file stays small; the uint8 crops are stored whole.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from crop_cases import CONFIGS, DEGENERATE, pattern_images, random_boxes, sha256  # noqa: E402

N_BOXES = {"256": 14, "128": 18}
K = 9


def _reference():
    ref = os.environ.get("PVNET_REFERENCE")
    if not ref or not os.path.isdir(ref):
        raise SystemExit("set PVNET_REFERENCE to a clean-pvnet checkout")
    sys.path.insert(0, ref)
    cfg = types.SimpleNamespace(tless=types.SimpleNamespace(
        pvnet_input_scale=(256, 256), scale_train_ratio=(1.8, 2.4), scale_ratio=2.4, box_train_ratio=(1.0, 1.2),
        box_ratio=1.2, rot=360., ratio=0.8))
    config = types.ModuleType("lib.config")
    config.cfg, config.args = cfg, None
    sys.modules["lib.config"] = config
    aug = types.ModuleType("imgaug")
    aug.augmenters = types.ModuleType("imgaug.augmenters")
    for name in ("Sequential", "Sometimes", "GaussianBlur", "AdditiveGaussianNoise", "Add", "Multiply",
                 "ContrastNormalization", "AddToHueAndSaturation"):
        setattr(aug.augmenters, name, lambda *a, **k: None)      # built at import by tless_train_utils, never called
    sys.modules["imgaug"], sys.modules["imgaug.augmenters"] = aug, aug.augmenters
    from lib.utils.tless import tless_test_utils, tless_config, tless_pvnet_utils
    from lib.utils import data_utils
    return tless_test_utils, tless_config, tless_pvnet_utils, data_utils


def main():
    tu, tc, tp, du = _reference()
    rng = np.random.default_rng(20261016)
    params = rng.integers(1, 1 << 16, (2, 3, 4))
    img = pattern_images(params)
    res = {"img_params": params}
    for name, ((w, h), scale_ratio, box_ratio) in CONFIGS.items():
        tc.scale_ratio, tc.box_ratio = scale_ratio, box_ratio
        tp.input_scale = np.array([w, h])
        boxes = np.concatenate([random_boxes(rng, N_BOXES[name] - len(DEGENERATE)), DEGENERATE])
        index = rng.integers(0, len(img), len(boxes)).astype(np.int32)
        kpt = rng.uniform(-20, max(w, h) + 20, (len(boxes), K, 2)).astype(np.float32)
        crops, digests, centers, scales, uncrop = [], [], [], [], []
        for b, i, kp in zip(boxes, index, kpt):
            orig, inp, center, scale = tu.pvnet_transform(img[i], list(b))
            assert inp.dtype == np.float32 and orig.dtype == np.uint8 and center.dtype == np.float32
            crops.append(orig)
            digests.append(sha256(inp))
            centers.append(center)
            scales.append(float(scale))
            trans_inv = du.get_affine_transform(center, np.float64(scale), 0, [w, h], inv=1)
            uncrop.append(du.affine_transform(kp, trans_inv))
        res.update({f"{name}_boxes": boxes, f"{name}_index": index, f"{name}_kpt": kpt,
                    f"{name}_crop": np.stack(crops), f"{name}_inp_sha256": np.array(digests),
                    f"{name}_center": np.stack(centers), f"{name}_scale": np.array(scales, np.float64),
                    f"{name}_uncrop": np.stack(uncrop), f"{name}_config": np.array([w, h, scale_ratio, box_ratio])})
    np.savez_compressed(os.path.join(HERE, "tless_crop.npz"), **res)
    print({k: v.shape for k, v in res.items()})


if __name__ == "__main__":
    main()
