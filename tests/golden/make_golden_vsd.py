"""Writes tests/golden/vsd.npz: the VSD error of clean-pvnet's own `lib/utils/vsd` code (vsd_utils.vsd with the 'step'
cost, misc.depth_im_to_dist_im, visibility.estimate_visib_mask_gt / _est, called as Evaluator.vsd_metric calls them,
lib/evaluators/tless_test/pvnet.py:66-105) on seeded synthetic depth images.

    PVNET_REFERENCE=/path/to/clean-pvnet python tests/golden/make_golden_vsd.py

vsd_utils imports `renderer`, which imports glumpy at module level; a stub module stands in for it, since VSD itself
never renders.  The cases cover zeros in every image, empty unions, distances straddling delta and tau, and non-square K.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
H, W = 40, 56
DELTA, TAU = 15, 20                 # lib/utils/tless/tless_config.py


def _reference():
    ref = os.environ.get("PVNET_REFERENCE")
    if not ref or not os.path.isdir(ref):
        raise SystemExit("set PVNET_REFERENCE to a clean-pvnet checkout")
    sys.path.insert(0, ref)
    sys.modules["lib.utils.vsd.renderer"] = types.ModuleType("lib.utils.vsd.renderer")   # no glumpy
    from lib.utils.vsd import vsd_utils
    return vsd_utils


def _cases(rng):
    Ks = [np.array([[1075.65, 0, 27.3], [0, 1073.90, 19.8], [0, 0, 1]]),        # T-LESS-like focal lengths
          np.array([[572.4114, 0, 25.0], [0, 573.57043, 21.5], [0, 0, 1]]),
          np.array([[300.0, 0, 31.7], [0, 150.0, 11.2], [0, 0, 1]])]            # strongly non-square
    for ci in range(12):
        K = Ks[ci % 3]
        test = (rng.integers(6000, 9000, (H, W)) * 0.1).astype(np.float32)   # load_depth(path) * 0.1 of a uint16 image
        test[rng.random((H, W)) < 0.15] = 0
        kind = ci % 4
        if kind == 0:      # surfaces near the scene: differences straddle delta
            gt = test + rng.uniform(-2 * DELTA, 2 * DELTA, (H, W)).astype(np.float32)
            est = test + rng.uniform(-2 * DELTA, 2 * DELTA, (H, W)).astype(np.float32)
        elif kind == 1:    # estimate within a few tau of the ground truth: |dist_gt - dist_est| straddles tau
            gt = test + rng.uniform(-DELTA, DELTA, (H, W)).astype(np.float32)
            off = rng.choice([-1, 1], (H, W)) * rng.uniform(TAU - 0.05, TAU + 0.05, (H, W))
            est = gt + np.where(rng.random((H, W)) < 0.2, off, rng.uniform(-1, 1, (H, W))).astype(np.float32)
            gt[rng.random((H, W)) < 0.2] = 0                             # one background for both renders
            est[gt == 0] = 0
        elif kind == 2:    # values on the thresholds' grid, so ties happen in float32
            gt = test + rng.integers(-4, 5, (H, W)).astype(np.float32) * 5
            est = gt + rng.integers(-6, 7, (H, W)).astype(np.float32) * 5
        else:              # an object silhouette in front of / behind the scene
            gt = np.where(rng.random((H, W)) < 0.5, test - 30, test + 30).astype(np.float32)
            est = np.roll(gt, 3, axis=1)
        if kind != 1:
            for img in (gt, est):
                img[rng.random((H, W)) < 0.3] = 0                        # background of the renders
        gt[gt < 0] = 0
        est[est < 0] = 0
        yield K, test, gt.astype(np.float32), est.astype(np.float32)
    K = Ks[0]
    z = np.zeros((H, W), np.float32)
    yield K, z.copy(), z.copy(), z.copy()                                 # every image empty: empty union, e = 1
    test = np.full((H, W), 700.0, np.float32)
    yield K, test, z.copy(), z.copy()                                     # nothing rendered: empty union
    yield K, z.copy(), test.copy(), test.copy()                           # no test depth: nothing visible, e = 1
    yield K, test, test.copy(), z.copy()                                  # estimate renders nothing: e = 1


def main():
    vsd_utils = _reference()
    rng = np.random.default_rng(20261016)
    Ks, tests, gts, ests, es = [], [], [], [], []
    for K, test, gt, est in _cases(rng):
        dist_test = vsd_utils.misc.depth_im_to_dist_im(test, K)
        dist_gt = vsd_utils.misc.depth_im_to_dist_im(gt, K)
        dist_est = vsd_utils.misc.depth_im_to_dist_im(est, K)
        visib_gt = vsd_utils.visibility.estimate_visib_mask_gt(dist_test, dist_gt, DELTA)
        e = vsd_utils.vsd(dist_est, dist_gt, dist_test, visib_gt, DELTA, TAU, 'step')
        Ks.append(K); tests.append(test); gts.append(gt); ests.append(est); es.append(float(e))
    np.savez_compressed(os.path.join(HERE, "vsd.npz"), K=np.stack(Ks), depth_test=np.stack(tests), depth_gt=np.stack(gts),
                        depth_est=np.stack(ests), e=np.array(es, np.float64), delta=DELTA, tau=TAU)
    print("e =", np.round(es, 4))


if __name__ == "__main__":
    main()
