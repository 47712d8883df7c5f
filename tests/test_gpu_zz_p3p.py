"""GPU: the device launch of the P3P initialisation (pvb_uncertainty_pnp_init, csrc/pnp.cu p3p_start_kernel:
p3p_start, one thread per problem).

Its arithmetic (csrc/p3p_core.cuh) is pinned against cv2.solvePnP on the CPU by tests/test_p3p_host_core.py; what is checked
here is the launch, the point selection on the device and the memory layout (first GPU run: the round-1 driver, passed)."""
import numpy as np
import pytest
import torch

from util import pnp_case

pytestmark = pytest.mark.gpu


def test_device_p3p_matches_opencv(pvb):
    cv2 = pytest.importorskip("cv2")
    cases = [pnp_case(2000 + s, pn=9, noise=[0.0, 1.0, 5.0][s % 3]) for s in range(200)]
    f = lambda i: torch.from_numpy(np.stack([c[i] for c in cases])).cuda()   # noqa: E731
    init = pvb.p3p_init_batch(f(0), f(2), f(1), f(3)).cpu().numpy()
    bad = 0
    for c, rt in zip(cases, init):
        uv, p3, W, K = c[:4]
        idx = np.argsort(W[:, 0] + W[:, 1], kind="stable")[-4:]
        ok, rvec, tvec = cv2.solvePnP(np.expand_dims(p3[idx], 0), np.expand_dims(uv[idx], 0), K, np.zeros((8, 1)), None, None, False,
                                      flags=cv2.SOLVEPNP_P3P)
        if not (np.isfinite(rvec).all() and np.isfinite(tvec).all()):
            assert np.isnan(rt).all()
            continue
        d = max(np.abs(cv2.Rodrigues(rt[:3].reshape(3, 1))[0] - cv2.Rodrigues(rvec)[0]).max(), np.abs(rt[3:] - tvec.ravel()).max())
        bad += d > 1e-6
    assert bad <= 1                                   # a tie of OpenCV's own ranking (tests/test_p3p_host_core.py)


def test_device_p3p_feeds_the_refinement(pvb):
    """init_rt=None: P3P on the device, then the LM refinement; the pose must be the one the refinement reaches from OpenCV's
    P3P pose (same optimum), for a batch with one shared model and camera."""
    cv2 = pytest.importorskip("cv2")
    import pnp_oracle as po
    base = pnp_case(3000, pn=9)
    cases = []
    for s in range(8):
        c = pnp_case(3001 + s, pn=9, noise=1.0)
        R = po.rodrigues(c[5][:3])
        cam = base[1] @ R.T + c[5][3:]
        uv = np.stack([base[3][0, 0] * cam[:, 0] / cam[:, 2] + base[3][0, 2], base[3][1, 1] * cam[:, 1] / cam[:, 2] + base[3][1, 2]], 1)
        uv += np.random.default_rng(3100 + s).normal(size=uv.shape)
        cases.append((uv, c[2]))
    uv = torch.from_numpy(np.stack([c[0] for c in cases])).cuda()
    W = torch.from_numpy(np.stack([c[1] for c in cases])).cuda()
    rt = pvb.uncertainty_pnp_batch(uv, W, torch.from_numpy(base[1]).cuda(), torch.from_numpy(base[3]).cuda()).cpu().numpy()
    for (u, w), got in zip(cases, rt):
        idx = np.argsort(w[:, 0] + w[:, 1], kind="stable")[-4:]
        _, rvec, tvec = cv2.solvePnP(np.expand_dims(base[1][idx], 0), np.expand_dims(u[idx], 0), base[3], np.zeros((8, 1)), None, None,
                                     False, flags=cv2.SOLVEPNP_P3P)
        want = po.uncertainty_pnp(u, base[1], w, base[3], np.concatenate([rvec, tvec], 0).reshape(6))
        assert np.abs(got - want).max() < 2e-4
