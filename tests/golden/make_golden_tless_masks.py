"""Writes tests/golden/tless_masks.npz: T-LESS's instance label maps, pixel counts and boxes as clean-pvnet's own
lib/datasets/tless code builds them, on the seeded mm depth stacks of tests/tless_mask_cases.py.

    PVNET_REFERENCE=/path/to/clean-pvnet python tests/golden/make_golden_tless_masks.py

Per image it runs what get_mask does (handle_test_data.py:116-128): opengl_renderer.render(model, pose, K, w, h), then
update_mask into an int16 label map and a depth map of 10, and np.sum(depth != 0) for pixel_num.pkl; then what
test_to_coco takes from the written mask (:42-52): np.sum(mask == mask_id) and cv2.boundingRect / area of that mask.
`lib.datasets.tless.opengl_backend` imports glumpy and needs a GL context, so a stub takes its place that returns the
case's fp32 mm depth for the instance (after checking the size, clip planes and mode render passes it);
opengl_renderer.render divides it by 1000 as it does for the real renderer.  `lib.config`, which tless_config imports
and which parses the command line, is a stub too, and so is the `lib.datasets` package, whose __init__ builds the data
loaders.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from tless_mask_cases import cases  # noqa: E402


def _reference():
    ref = os.environ.get("PVNET_REFERENCE")
    if not ref or not os.path.isdir(ref):
        raise SystemExit("set PVNET_REFERENCE to a clean-pvnet checkout")
    sys.path.insert(0, ref)
    config = types.ModuleType("lib.config")
    config.cfg = types.SimpleNamespace(tless=types.SimpleNamespace(      # read by tless_config at import, unused here
        pvnet_input_scale=(256, 256), scale_train_ratio=(1.8, 2.4), scale_ratio=2.4, box_train_ratio=(1.0, 1.2),
        box_ratio=1.2))
    sys.modules["lib.config"] = config
    backend = types.ModuleType("lib.datasets.tless.opengl_backend")

    def render(model, im_size, K, R, t, clip_near=100, clip_far=2000, mode='rgb+depth', **kwargs):
        d = model["depth_mm"]
        assert list(im_size) == [d.shape[1], d.shape[0]] and (clip_near, clip_far, mode) == (10, 10000, 'depth')
        return d.copy()
    backend.render = render
    sys.modules["lib.datasets.tless.opengl_backend"] = backend
    # lib/datasets/__init__.py builds the data loaders (and reads cfg) on import; only the tless files are needed
    datasets = types.ModuleType("lib.datasets")
    datasets.__path__ = [os.path.join(ref, "lib", "datasets")]
    sys.modules["lib.datasets"] = datasets
    import lib.datasets.tless as tless_pkg
    tless_pkg.opengl_backend = backend
    from lib.datasets.tless import opengl_renderer, handle_test_data
    return opengl_renderer, handle_test_data


def main():
    import cv2
    opengl_renderer, handle_test_data = _reference()
    K = np.array([[1075.65, 0, 367.07], [0, 1073.90, 247.72], [0, 0, 1]])
    pose = np.concatenate([np.eye(3), np.array([[0.0], [0.0], [0.7]])], axis=1)
    out = {}
    for ci, (name, depth_mm, obj_ids) in enumerate(cases()):
        m, h, w = depth_mm.shape
        mask_map = np.zeros(shape=[h, w], dtype=np.int16)
        depth_map = 10 * np.ones(shape=[h, w], dtype=np.float32)
        a_pixel_nums = []
        for instance_id in range(m):
            depth = opengl_renderer.render({"depth_mm": depth_mm[instance_id]}, pose, K, w, h)
            handle_test_data.update_mask(depth, w, mask_map, depth_map, int(obj_ids[instance_id]), instance_id)
            a_pixel_nums.append(np.sum(depth != 0))
        pixel_num, bbox, area = [], [], []
        for instance_id in range(m):
            mask_ = (mask_map == int(obj_ids[instance_id]) * 1000 + instance_id).astype(np.uint8)
            pixel_num.append(np.sum(mask_))
            bbox.append(cv2.boundingRect(mask_))
            area.append(int(np.sum(mask_.astype(np.uint8))))
        out[f"c{ci}_name"] = np.array(name)
        out[f"c{ci}_depth"] = depth_mm
        out[f"c{ci}_obj_ids"] = np.asarray(obj_ids, np.int64)
        out[f"c{ci}_label"] = mask_map
        out[f"c{ci}_a_pixel_num"] = np.array(a_pixel_nums, np.int64)
        out[f"c{ci}_pixel_num"] = np.array(pixel_num, np.int64)
        out[f"c{ci}_bbox"] = np.array(bbox, np.int64).reshape(m, 4)
        out[f"c{ci}_area"] = np.array(area, np.int64)
        print(name, depth_mm.shape, "a", a_pixel_nums, "p", pixel_num)
    out["n_cases"] = np.array(len(cases()))
    np.savez_compressed(os.path.join(HERE, "tless_masks.npz"), **out)


if __name__ == "__main__":
    main()
