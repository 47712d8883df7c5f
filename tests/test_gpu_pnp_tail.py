"""GPU: the fused un_pnp tail (`uncertainty_pnp_from_votes`, the fp32 instantiation of csrc/pnp.cu pnp_batch_kernel) and
the batched refinement (`uncertainty_pnp_batch`, its fp64 instantiation) against real Ceres and OpenCV, through
tests/golden/ceres_pnp_fp32.npz (tests/golden/make_golden_ceres_fp32.py; the CPU side, tests/test_ceres_golden.py and tests/test_p3p_host_core.py, checks
that the oracle and the host builds of pnp_core.cuh / p3p_core.cuh follow the same fixture).

The fixture's inputs are fp32 keypoints, fp32 covariances and the fp32 weights cov_to_weights makes of them -- exactly what
the fused entry takes -- at pn = 9 and 17 with one model and camera for the batch (stride 0), at pn = 31..64 with a model
and a camera per problem (the strides), with zero-weight and negative-key keypoints, skipped images and pn = 3 / 4.  Batches
of 1, 3, 5 and 130 problems leave the last CTA partly filled.

Bar (as test_gpu_pnp.py::test_kernel_follows_real_ceres): on problems Ceres can be followed on (`stable`) the same stop
reason, the same iteration count and the pose within 1e-9 for at least 97 %; otherwise the pose within 2e-4, the slack of
Ceres' function_tolerance."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ceres_pnp_fp32.npz"))
NF = len(F["pn"])


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def groups(kinds=None, pns=None):
    """(kind, pn, fixture indices) for every set and point count."""
    for kind in ("prod9", "prod17", "wide", "zeros", "skipped", "small"):
        for pn in np.unique(F["pn"][F["kind"] == kind]):
            if (kinds is None or kind in kinds) and (pns is None or pn in pns):
                yield kind, int(pn), np.nonzero((F["kind"] == kind) & (F["pn"] == pn))[0]


def inputs(idx, pn):
    """kpt [n,pn,2] fp32, cov [n,pn,2,2] fp32, weights [n,pn,3] fp32, model, camera: [pn,3] / [3,3] for a shared set
    (stride 0), [n,pn,3] / [n,3,3] otherwise."""
    shared = bool(F["shared"][idx].all())
    model = F["pts3d"][idx[0], :pn] if shared else F["pts3d"][idx, :pn]
    cam = F["K"][idx[0]] if shared else F["K"][idx]
    return t(F["kpt2d"][idx, :pn]), t(F["cov"][idx, :pn]), t(F["wgt2d"][idx, :pn]), t(model), t(cam)


def expected(i, start):
    reason = int(F[start + "reason"][i])
    return int(F[start + "iteration_summaries"][i]) - (0 if reason in (2, 3) else 1), reason


class Tally:
    """Counts the followable problems and those followed iteration for iteration; checks every pose against its bar."""

    def __init__(self):
        self.same = self.total = 0

    def check(self, i, start, rt, info, where):
        want = F[start + "result_rt"][i]
        if not F[start + "stable"][i]:
            assert 1 <= info[1] <= 6, (where, i)
            return
        self.total += 1
        if (int(info[0]), int(info[1])) == expected(i, start):
            self.same += 1
            assert np.abs(rt - want).max() < 1e-9, (where, i, np.abs(rt - want).max())
        else:
            assert np.abs(rt - want).max() < 2e-4, (where, i, np.abs(rt - want).max())

    def assert_bar(self, at_least):
        assert self.total >= at_least and self.same >= 0.97 * self.total, (self.same, self.total)


def bits(x):
    return x.contiguous().view(torch.int64)


@pytest.mark.parametrize("start", ["", "p3ps_"])
def test_fused_kernel_follows_ceres(pvb, start):
    """The fused entry with `weights` and an explicit start (the perturbed truth, or OpenCV's P3P pose on the stable top
    four) against Ceres from the same start, every set; the fp64 instantiation on the same data gives identical bits; the problem's
    place in the batch (n = 1, 3, 5, 130, partly filled CTAs) changes nothing."""
    tally = Tally()
    init_all = F["init_rt"] if start == "" else F["p3ps_rt"]
    for kind, pn, idx in groups():
        if start and pn < 4:
            continue
        kpt, _, w, model, cam = inputs(idx, pn)
        init = t(init_all[idx])
        rt, info = pvb.uncertainty_pnp_from_votes(kpt, None, model, cam, init_rt=init, weights=w, return_info=True)
        rt_np, info_np = rt.cpu().numpy(), info.cpu().numpy()
        for j, i in enumerate(idx):
            tally.check(i, start, rt_np[j], info_np[j], (kind, pn))
        # the fp64 instantiation (double inputs, the same values) must give the same bits, incl. pn > 32
        rt2, info2 = pvb.uncertainty_pnp_batch(kpt.double(), w.double(), model, cam, init, return_info=True)
        assert torch.equal(bits(rt2), bits(rt)) and torch.equal(info2, info), (kind, pn)
        # partly filled CTAs and many problems per launch: each row is the same as in the whole-set batch
        for n in (1, 3, 5, 130):
            sel = np.arange(n) % len(idx)
            k_, _, w_, m_, c_ = inputs(idx[sel], pn)
            rt_n, info_n = pvb.uncertainty_pnp_from_votes(k_, None, m_, c_, init_rt=t(init_all[idx[sel]]), weights=w_,
                                                         return_info=True)
            assert torch.equal(bits(rt_n), bits(rt[sel])) and torch.equal(info_n, info[sel]), (kind, pn, n)
    tally.assert_bar(215 if start else 228)


@pytest.mark.parametrize("pn", [9, 17, 33, 64])
def test_whole_tail_from_var(pvb, pn):
    """cov in, no start: the fused kernel's weights are the fixture's bit for bit, its P3P pose (`init_out`) is OpenCV's on
    the stable top four (to 1e-6, except where the fourth point cannot tell two candidates apart), p3p_init_batch gives
    the same bits, and the result follows Ceres started from OpenCV's pose."""
    import cv2
    tally, ties, followable = Tally(), [], 0
    for kind, _, idx in groups(kinds=("prod9", "prod17", "wide", "zeros"), pns=(pn,)):
        followable += int(F["p3ps_stable"][idx].sum())
        kpt, cov, w, model, cam = inputs(idx, pn)
        rt, info, init_out, w_out = pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, return_info=True, return_aux=True)
        assert torch.equal(w_out.view(torch.int32), w.view(torch.int32)), kind
        assert torch.equal(bits(pvb.p3p_init_batch(kpt, w, model, cam)), bits(init_out)), kind
        # from the same start, the weights it derived itself and the fixture's fp32 weights give the same bits
        rt_w = pvb.uncertainty_pnp_from_votes(kpt, None, model, cam, init_rt=init_out, weights=w)
        assert torch.equal(bits(rt_w), bits(rt)), kind
        rt, info, init_out = rt.cpu().numpy(), info.cpu().numpy(), init_out.cpu().numpy()
        for j, i in enumerate(idx):
            want = F["p3ps_rt"][i]
            if not np.isfinite(want).all():
                assert np.isnan(init_out[j]).all() and np.isnan(rt[j]).all(), (kind, i)
                continue
            rot = lambda a: cv2.Rodrigues(np.ascontiguousarray(a[:3]).reshape(3, 1))[0]   # noqa: E731
            d = max(np.abs(rot(init_out[j]) - rot(want)).max(), np.abs(init_out[j, 3:] - want[3:]).max())
            if d > 1e-6:                       # a tie of OpenCV's own ranking: Ceres from the other root is not comparable
                ties.append(i)
                continue
            tally.check(i, "p3ps_", rt[j], info[j], (kind, pn))
    assert len(ties) <= 1, ties
    assert followable >= {9: 80, 17: 80, 33: 8, 64: 8}[pn]
    tally.assert_bar(followable - len(ties))


def test_skipped_image(pvb):
    """An image the voting layer skipped (kpt = 0, cov = 0): every weight is 0 and the four image points coincide.
    OpenCV's P3P answers (True, rvec = 0, tvec = NaN) and Ceres refuses that start (FAILURE, pose unchanged); the device P3P
    finds no admissible pose and returns all-NaN, and the refinement stops at once on it (gradient test, 0 iterations).
    Either way the translation is NaN; only the rotation of the failed pose differs (0 in the reference, NaN here).  From a
    finite start both sides stop at once with the pose untouched: every residual is 0."""
    for _, pn, idx in groups(kinds=("skipped",)):
        kpt, cov, w, model, cam = inputs(idx, pn)
        rt, info, init_out, _ = pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, return_info=True, return_aux=True)
        rt, info, init_out = rt.cpu().numpy(), info.cpu().numpy(), init_out.cpu().numpy()
        for j, i in enumerate(idx):
            ref_init, ref_rt = F["p3p_rt"][i], F["p3p_result_rt"][i]
            assert (ref_init[:3] == 0).all() and np.isnan(ref_init[3:]).all() and F["p3p_reason"][i] == 6    # the reference
            assert np.array_equal(ref_rt, ref_init, equal_nan=True)
            assert np.isnan(init_out[j]).all() and np.isnan(rt[j]).all() and tuple(info[j]) == (0, 1)       # this project
        init = t(F["init_rt"][idx])
        rt, info = pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, init_rt=init, return_info=True)
        for j, i in enumerate(idx):
            assert (int(info[j, 0]), int(info[j, 1])) == expected(i, "") == (0, 1)
            assert np.array_equal(rt[j].cpu().numpy(), F["result_rt"][i]) and np.array_equal(F["result_rt"][i], F["init_rt"][i])


def test_nan_and_zero_covariances(pvb):
    """Keypoints whose covariance is NaN, all zero or has cov[0,0] < 1e-6 get weight 0 in the fused kernel as in the
    reference; a whole image of NaN or zero covariances keeps its keypoints, P3P runs on the last four and the refinement
    stops at once on that pose (every residual weighted 0), as Ceres does from OpenCV's pose."""
    for _, pn, idx in groups(kinds=("zeros",)):
        kpt, cov, w, model, cam = inputs(idx, pn)
        rt, info, init_out, w_out = pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, return_info=True, return_aux=True)
        assert torch.equal(w_out, w)
        c = F["cov"][idx, :pn]
        dead = np.isnan(c).any((2, 3)) | (c[..., 0, 0] < 1e-6)
        assert dead.any(1).all() and not w_out.cpu().numpy()[dead].any()
        whole = dead.all(1)
        assert whole.sum() == 4
        info, rt, init_out = info.cpu().numpy(), rt.cpu().numpy(), init_out.cpu().numpy()
        for j in np.nonzero(whole)[0]:
            i = idx[j]
            assert F["idx_stable"][i].tolist() == list(range(pn - 4, pn)) and tuple(info[j]) == (0, 1)
            assert np.array_equal(rt[j], init_out[j]) and expected(i, "p3ps_") == (0, 1)
            assert np.abs(rt[j] - F["p3ps_result_rt"][i]).max() < 1e-6


def test_four_and_three_points(pvb):
    """pn = 4: P3P takes every point (three solve, the fourth picks the root) and the fused tail refines on all four, as
    Ceres does from that start (the reference's un_pnp_utils.uncertainty_pnp returns the P3P pose itself at pn = 4, and so
    does its twin clean_pvnet_b200.un_pnp.uncertainty_pnp).  pn = 3: no P3P start, so an `init_rt` is required, and the
    refinement follows Ceres from it."""
    import cv2
    (_, _, i4), = groups(kinds=("small",), pns=(4,))
    kpt, cov, w, model, cam = inputs(i4, 4)
    rt, info, init_out, _ = pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, return_info=True, return_aux=True)
    rt, info, init_out = rt.cpu().numpy(), info.cpu().numpy(), init_out.cpu().numpy()
    tally = Tally()
    for j, i in enumerate(i4):
        assert sorted(F["idx_stable"][i].tolist()) == [0, 1, 2, 3]
        want = F["p3ps_rt"][i]
        rot = lambda a: cv2.Rodrigues(np.ascontiguousarray(a[:3]).reshape(3, 1))[0]   # noqa: E731
        assert np.abs(rot(init_out[j]) - rot(want)).max() < 1e-6 and np.abs(init_out[j, 3:] - want[3:]).max() < 1e-6, i
        tally.check(i, "p3ps_", rt[j], info[j], 4)
    tally.assert_bar(8)
    (_, _, i3), = groups(kinds=("small",), pns=(3,))
    kpt, cov, w, model, cam = inputs(i3, 3)
    with pytest.raises(RuntimeError):
        pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam)
    rt, info = pvb.uncertainty_pnp_from_votes(kpt, cov, model, cam, init_rt=t(F["init_rt"][i3]), return_info=True)
    rt, info = rt.cpu().numpy(), info.cpu().numpy()
    tally = Tally()
    for j, i in enumerate(i3):
        tally.check(i, "", rt[j], info[j], 3)
    tally.assert_bar(8)


def test_more_than_64_points_is_refused(pvb):
    """The fused kernel stages a problem in shared memory sized for 64 points: pn = 65 is an error, not a silent overrun;
    pn = 64 runs (test_fused_kernel_follows_ceres)."""
    kpt = torch.zeros((2, 65, 2), device="cuda")
    w = torch.ones((2, 65, 3), device="cuda")
    model = torch.zeros((65, 3), dtype=torch.float64, device="cuda")
    cam = torch.eye(3, dtype=torch.float64, device="cuda")
    init = torch.zeros((2, 6), dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError, match="pn must be in"):
        pvb.uncertainty_pnp_from_votes(kpt, None, model, cam, init_rt=init, weights=w)
    with pytest.raises(RuntimeError, match="pn must be in"):
        pvb.uncertainty_pnp_from_votes(kpt, torch.zeros((2, 65, 2, 2), device="cuda"), model, cam)
