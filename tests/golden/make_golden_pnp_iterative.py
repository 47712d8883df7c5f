"""Writes tests/golden/pnp_iterative.npz: cv2.solvePnP(..., SOLVEPNP_ITERATIVE) called as lib/utils/pvnet/
pvnet_pose_utils.py:5-38 calls it, on 240 followable problems of tests/pnp_iter_cases.py (pn in {6, 7, 9, 17, 33, 64},
noise 0-20 px, vote outliers, rotations near 0 and pi, per-problem intrinsics), so the GPU test does not depend on the
OpenCV installed next to the GPU.  A problem is kept when OpenCV re-run on its image points scaled by (1 + 1e-13) moves by
at most 1e-8 (the pin's followability rule).  Ragged layout: problem i's points are rows off[i]:off[i+1].

    python tests/golden/make_golden_pnp_iterative.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from pnp_iter_cases import cases, opencv_pnp, rel_diff  # noqa: E402


def main():
    import cv2
    keep = []
    for uv, X, K in cases(260, seed0=100000):
        rt = opencv_pnp(X, uv, K)
        if rel_diff(rt, opencv_pnp(X, uv * (1 + 1e-13), K)) <= 1e-8:
            keep.append((uv, X, K, rt))
    keep = keep[:240]
    assert len(keep) == 240
    pn = np.array([k[0].shape[0] for k in keep], np.int32)
    rt = np.stack([k[3] for k in keep])
    pose = np.stack([np.concatenate([cv2.Rodrigues(r[:3])[0], r[3:, None]], 1) for r in rt])
    np.savez_compressed(os.path.join(HERE, "pnp_iterative.npz"),
                        off=np.concatenate([[0], np.cumsum(pn)]).astype(np.int64), pn=pn,
                        pts2d=np.concatenate([k[0] for k in keep]), pts3d=np.concatenate([k[1] for k in keep]),
                        K=np.stack([k[2] for k in keep]), rt=rt, pose=pose, opencv_version=np.array(cv2.__version__))


if __name__ == "__main__":
    main()
