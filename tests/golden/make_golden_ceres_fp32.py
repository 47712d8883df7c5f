#!/usr/bin/env python
"""Generates tests/golden/ceres_pnp_fp32.npz: uncertainty-PnP problems whose inputs are exactly what the fused un_pnp tail
(`uncertainty_pnp_from_votes`, csrc/pnp.cu pnp_fused_kernel) sees -- fp32 keypoints, fp32 covariances and the fp32 weights
cov_to_weights derives from them, float64 model points and intrinsics -- solved by REAL Ceres 2.0 (the reference's prebuilt
libceres + its unmodified uncertainty_pnp.cpp, built by oracle/build_ceres_ref.py) and started from OpenCV's P3P pose as
un_pnp_utils.py:25-31 computes it.  CPU only; needs /root/reference:

    python tests/golden/make_golden_ceres_fp32.py

Sets (`kind`):
    prod9    pn = 9, one model and one camera for the set, 64 problems (the evaluator's LINEMOD shape)
    prod17   pn = 17, shared model and camera, 64 problems (T-LESS)
    wide     pn in {31, 32, 33, 48, 63, 64}, 8 each, a model and a camera per problem
    zeros    pn in {9, 17}, 16 each: zero-weight keypoints (cov[0,0] < 1e-6, NaN, all zero), fewer than four positive keys,
             negative keys wxx + wxy < 0, whole images of zero or NaN covariances
    skipped  pn in {9, 17}, 2 each: kpt = 0 and cov = 0, as the voting layer delivers an image it skipped
    small    pn in {3, 4}, 8 each, a model and a camera per problem (pn = 3 has no P3P start)

Per problem, three Ceres solves, each recorded as in ceres_pnp.npz (result, stop reason, #iteration summaries, costs,
`sensitivity` = how far the result moves when started from init*(1+1e-13), `stable` = below 1e-10):
    (no prefix)  started from `init_rt`, the true pose perturbed
    p3p_         started from `p3p_rt`  = cv2.solvePnP(P3P) on np.argsort(wxx + wxy)[-4:], the reference's own start
                 (numpy's default sort kind; `idx_default`)
    p3ps_        started from `p3ps_rt` = the same on np.argsort(..., kind="stable")[-4:] (`idx_stable`), the rule
                 p3p_select4 implements.  The two index sets differ only among tied keys.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import build_ceres_ref as ceres  # noqa: E402
from util import cov_to_weights_f32, pnp_case  # noqa: E402

PN_MAX = 64
LINEMOD_K = np.array([[572.4114, 0, 325.2611], [0, 573.57043, 242.04899], [0, 0, 1.0]])


def project(model, rt, K):
    import cv2
    R = cv2.Rodrigues(np.asarray(rt[:3], np.float64).reshape(3, 1))[0]
    c = model @ R.T + rt[3:]
    return np.stack([K[0, 0] * c[:, 0] / c[:, 2] + K[0, 2], K[1, 1] * c[:, 1] / c[:, 2] + K[1, 2]], 1)


def random_cov(rng, pn):
    A = rng.normal(size=(pn, 2, 2))
    return (A @ A.transpose(0, 2, 1) * rng.uniform(0.5, 4, size=(pn, 1, 1)) + 0.1 * np.eye(2)).astype(np.float32)


def problem(seed, pn, model=None, K=None, noise=None):
    """(kpt fp32 [pn,2], cov fp32 [pn,2,2], pts3d [pn,3], K [3,3], init_rt [6]) in the util.pnp_case geometry; the keypoints
    are the projection of `model` with the case's true pose under `K`, plus noise."""
    rng = np.random.default_rng(10_000 + seed)
    far = seed % 3 == 0
    c = pnp_case(seed, pn=pn, pert=(0.3, 0.1) if far else (0.05, 0.02))
    model = c[1] if model is None else model
    K = c[3] if K is None else K
    noise = [0.5, 1.0, 2.0][seed % 3] if noise is None else noise
    uv = project(model, c[5], K) + rng.normal(size=(pn, 2)) * noise
    return uv.astype(np.float32), random_cov(rng, pn), model, K, c[4]


def own_camera(seed):
    rng = np.random.default_rng(20_000 + seed)
    K = LINEMOD_K.copy()
    K[0, 0] *= rng.uniform(0.8, 1.25)
    K[1, 1] = K[0, 0] * rng.uniform(0.98, 1.02)
    K[0, 2] += rng.uniform(-20, 20)
    K[1, 2] += rng.uniform(-20, 20)
    return K


def negative_key_cov(rng):
    """A covariance whose inv(sqrtm) has wxx + wxy < 0: strongly correlated, cov[0,0] > cov[1,1]."""
    a, d = rng.uniform(2.0, 4.0), rng.uniform(0.4, 1.0)
    b = rng.uniform(0.93, 0.97) * np.sqrt(a * d)
    return np.array([[a, b], [b, d]], np.float32)


def problem_sets():
    sets = []
    base9, base17 = pnp_case(7100, pn=9), pnp_case(7200, pn=17)
    for s in range(64):
        sets.append(("prod9", True, problem(7101 + s, 9, base9[1], base9[3])))
    for s in range(64):
        sets.append(("prod17", True, problem(7201 + s, 17, base17[1], base17[3])))
    for pn in (31, 32, 33, 48, 63, 64):
        for s in range(8):
            seed = 7300 + 10 * pn + s
            sets.append(("wide", False, problem(seed, pn, K=own_camera(seed))))
    for pn in (9, 17):
        for s in range(16):
            seed = 7400 + 20 * pn + s
            kpt, cov, model, K, init = problem(seed, pn)
            rng = np.random.default_rng(30_000 + seed)
            perm = rng.permutation(pn)
            v = s % 8
            if v == 0:                                   # the cov[0,0] < 1e-6 guard, on either side of fp32(1e-6)
                cov[perm[0], 0, 0] = 5e-7
                cov[perm[1], 0, 0] = np.nextafter(np.float32(1e-6), np.float32(0))
            elif v == 1:                                 # a NaN entry, an all-zero covariance
                cov[perm[0], 0, 1] = np.nan
                cov[perm[1]] = 0.0
            elif v == 2:                                 # three positive keys: a zero key makes the top four
                cov[perm[3:]] = 0.0
            elif v == 3:                                 # one positive key
                cov[perm[1:]] = 0.0
            elif v == 4:                                 # negative keys rank below the zero-weight keypoints
                for j in perm[:3]:
                    cov[j] = negative_key_cov(rng)
                cov[perm[3:5]] = 0.0
            elif v == 5:                                 # two positive and two negative keys, the rest zero
                cov[perm[2:4]] = [negative_key_cov(rng) for _ in range(2)]
                cov[perm[4:]] = 0.0
            elif v == 6:                                 # every covariance NaN
                cov[:] = np.nan
            else:                                        # every covariance zero, keypoints real
                cov[:] = 0.0
            sets.append(("zeros", False, (kpt, cov, model, K, init)))
    for pn, base in ((9, base9), (17, base17)):
        for s in range(2):
            init = pnp_case(7500 + 10 * pn + s, pn=pn)[4]
            sets.append(("skipped", True, (np.zeros((pn, 2), np.float32), np.zeros((pn, 2, 2), np.float32), base[1], base[3], init)))
    for pn in (3, 4):
        for s in range(8):
            seed = 7600 + 10 * pn + s
            sets.append(("small", False, problem(seed, pn, K=own_camera(seed))))
    return sets


def solve(uv, p3, W, K, init):
    with np.errstate(all="ignore"):
        res, info, tr = ceres.solve(uv, p3, W, K, init)
        ent = ceres.reference_entry(uv, p3, W, K, init)
        res2, _, _ = ceres.solve(uv, p3, W, K, init * (1.0 + 1e-13))
    assert np.array_equal(res, ent, equal_nan=True)
    sens = np.abs(res - res2).max() if (np.isfinite(res).all() and np.isfinite(res2).all()) else np.inf
    return res, info, sens


def opencv_p3p(p3, uv, K, idx):
    import cv2
    ok, r, t = cv2.solvePnP(np.expand_dims(p3[idx], 0), np.expand_dims(uv[idx], 0), K, np.zeros((8, 1)), None, None, False,
                            flags=cv2.SOLVEPNP_P3P)
    return np.concatenate([np.asarray(r, np.float64).ravel(), np.asarray(t, np.float64).ravel()]), bool(ok)


def main():
    import cv2
    if ceres.build() is None:
        raise SystemExit("needs the reference checkout (/root/reference)")
    sets = problem_sets()
    n = len(sets)
    out = dict(kind=np.array([k for k, _, _ in sets]), shared=np.array([s for _, s, _ in sets]), pn=np.zeros(n, np.int32),
               kpt2d=np.zeros((n, PN_MAX, 2), np.float32), cov=np.zeros((n, PN_MAX, 2, 2), np.float32),
               wgt2d=np.zeros((n, PN_MAX, 3), np.float32), pts3d=np.zeros((n, PN_MAX, 3)), K=np.zeros((n, 3, 3)),
               init_rt=np.zeros((n, 6)), idx_default=np.full((n, 4), -1, np.int32), idx_stable=np.full((n, 4), -1, np.int32),
               p3p_rt=np.full((n, 6), np.nan), p3p_ok=np.zeros(n, bool), p3ps_rt=np.full((n, 6), np.nan),
               numpy_version=np.array(np.__version__), opencv_version=np.array(cv2.__version__))
    for p in ("", "p3p_", "p3ps_"):
        out.update({p + "result_rt": np.full((n, 6), np.nan), p + "reason": np.zeros(n, np.int32),
                    p + "termination_type": np.zeros(n, np.int32), p + "iteration_summaries": np.zeros(n, np.int32),
                    p + "unsuccessful": np.zeros(n, np.int32), p + "final_cost": np.zeros(n), p + "sensitivity": np.zeros(n),
                    p + "stable": np.zeros(n, bool)})

    def record(p, i, uv, p3, W, K, init):
        res, info, sens = solve(uv, p3, W, K, init)
        out[p + "result_rt"][i] = res
        out[p + "reason"][i], out[p + "termination_type"][i] = info["reason"], info["termination_type"]
        out[p + "iteration_summaries"][i], out[p + "unsuccessful"][i] = info["iteration_summaries"], info["unsuccessful_steps"]
        out[p + "final_cost"][i], out[p + "sensitivity"][i], out[p + "stable"][i] = info["final_cost"], sens, sens < 1e-10

    for i, (_, _, (kpt, cov, p3, K, init)) in enumerate(sets):
        pn = len(kpt)
        w = cov_to_weights_f32(cov)
        out["pn"][i] = pn
        out["kpt2d"][i, :pn], out["cov"][i, :pn], out["wgt2d"][i, :pn] = kpt, cov, w
        out["pts3d"][i, :pn], out["K"][i], out["init_rt"][i] = p3, K, init
        uv, W = kpt.astype(np.float64), w.astype(np.float64)          # what un_pnp_utils.py:21-24 makes of them
        record("", i, uv, p3, W, K, init)
        if pn < 4:
            continue
        key = W[:, 0] + W[:, 1]                                      # un_pnp_utils.py:25
        out["idx_default"][i], out["idx_stable"][i] = np.argsort(key)[-4:], np.argsort(key, kind="stable")[-4:]
        out["p3p_rt"][i], out["p3p_ok"][i] = opencv_p3p(p3, uv, K, out["idx_default"][i])
        out["p3ps_rt"][i], _ = opencv_p3p(p3, uv, K, out["idx_stable"][i])
        record("p3p_", i, uv, p3, W, K, out["p3p_rt"][i])
        record("p3ps_", i, uv, p3, W, K, out["p3ps_rt"][i])
    np.savez_compressed(os.path.join(HERE, "ceres_pnp_fp32.npz"), **out)
    print(f"numpy {np.__version__}, OpenCV {cv2.__version__}")
    for kind in ("prod9", "prod17", "wide", "zeros", "skipped", "small"):
        m = out["kind"] == kind
        ties = (out["idx_default"][m] != out["idx_stable"][m]).any(1).sum()
        print(f"{kind:8s} n={m.sum():3d} pn={sorted(set(out['pn'][m].tolist()))} stable={out['stable'][m].sum():3d} "
              f"p3p_stable={out['p3p_stable'][m].sum():3d} p3ps_stable={out['p3ps_stable'][m].sum():3d} "
              f"sort kinds differ={ties} reasons={np.bincount(out['reason'][m], minlength=7).tolist()}")


if __name__ == "__main__":
    main()
