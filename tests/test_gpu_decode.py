"""GPU: the fused front end of decode_keypoint (SURVEY.md section 8f row 1, resnet18.py:65-76).
Bar: the mask is bit-identical to torch.argmax(seg, 1) (ties -> first index, NaN -> maximal), and keypoints /
covariances are identical to the unfused path (torch.argmax + the operators) under the same seed."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _network_output(cfg, seed, classes=2, layout_noise=True):
    from clean_pvnet_b200 import synth
    mask, vertex, kp = synth.make_inputs(cfg, device="cuda", seed=seed, layout="planar")
    B, H, W, K, _ = vertex.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    seg = torch.randn((B, classes, H, W), generator=g, device="cuda") * 0.3
    seg[:, 1] += (mask.float() * 2 - 1) * 1.5          # class 1 = object
    ver_nchw = vertex.permute(0, 3, 4, 1, 2).reshape(B, 2 * K, H, W).contiguous()
    return {"seg": seg, "vertex": ver_nchw}


@pytest.mark.parametrize("classes", [2, 3, 5])
def test_mask_equals_torch_argmax(pvb, classes):
    out = _network_output("small", 31, classes)
    seg = out["seg"]
    seg[0, :, 3, 4:9] = 0.25                                   # exact ties -> first index
    seg[1, classes - 1, 5, 5] = float("nan")                   # NaN counts as the maximum
    seg[1, 0, 6, 6] = float("nan")
    seg[2, :, 7, 7] = float("nan")
    res = pvb.decode_keypoint(dict(out), un_pnp=False, seed=5)
    want = torch.argmax(seg, 1)
    assert res["mask"].dtype == torch.int64 and torch.equal(res["mask"], want)


@pytest.mark.parametrize("un_pnp", [False, True])
def test_fused_equals_unfused(pvb, un_pnp):
    out = _network_output("small", 32)
    a = pvb.decode_keypoint(dict(out), un_pnp=un_pnp, seed=9, fused=True)
    b = pvb.decode_keypoint(dict(out), un_pnp=un_pnp, seed=9, fused=False)
    assert torch.equal(a["mask"], b["mask"])
    assert torch.equal(a["kpt_2d"], b["kpt_2d"])
    if un_pnp:
        assert torch.equal(a["var"], b["var"])
        assert a["var"].shape == (3, 4, 2, 2)
    else:
        assert "var" not in a


def test_matches_reference_decode_flow(pvb):
    """Same flow written with the reference's operator names (what resnet18.py does), strided seg view included."""
    out = _network_output("small", 33, classes=2)
    big = torch.zeros(3, 4, 96, 128, device="cuda")
    big[:, ::2] = out["seg"]
    seg_view = big[:, ::2]                                     # non-contiguous class stride
    res = pvb.decode_keypoint({"seg": seg_view, "vertex": out["vertex"]}, un_pnp=True, seed=11)
    vertex = out["vertex"].permute(0, 2, 3, 1).view(3, 96, 128, 4, 2)
    mask = torch.argmax(out["seg"], 1)
    mean = pvb.ransac_voting_layer_v3(mask, vertex, 512, inlier_thresh=0.99, seed=11)
    kpt, var = pvb.estimate_voting_distribution_with_mean(mask, vertex, mean, seed=11)
    assert torch.equal(res["mask"], mask) and torch.equal(res["kpt_2d"], kpt) and torch.equal(res["var"], var)


def test_uncertainty_pnp_weights_match_reference_formula(pvb):
    """SURVEY 8f row 2: inv(sqrtm(cov)) weights vs the reference's own CPU code (evaluators/linemod/pvnet.py:118-130)."""
    import numpy as np
    import scipy.linalg
    out = _network_output("small", 34)
    res = pvb.decode_keypoint(dict(out), un_pnp=True, seed=13)
    var = res["var"].clone()
    var[0, 0] = 0.0                       # var[0,0] < 1e-6 -> zeros
    var[1, 1, 0, 1] = float("nan")        # NaN -> zeros
    got = pvb.uncertainty_pnp_weights(var).cpu().numpy()
    v = var.cpu().numpy()
    for b in range(v.shape[0]):
        cov_invs = []
        for vi in range(v.shape[1]):      # verbatim logic of the reference loop
            if v[b, vi, 0, 0] < 1e-6 or np.sum(np.isnan(v[b])[vi]) > 0:
                cov_invs.append(np.zeros([2, 2]).astype(np.float32))
            else:
                cov_invs.append(np.linalg.inv(scipy.linalg.sqrtm(v[b, vi])))
        want = np.asarray(cov_invs).reshape([-1, 4])[:, (0, 1, 3)]
        assert np.allclose(got[b], np.real(want), rtol=2e-4, atol=1e-6), (got[b], want)
    assert (got[0, 0] == 0).all() and (got[1, 1] == 0).all()


def _weights_f64(c):
    """inv(sqrtm(C)) of the symmetric part of fp32 covariances c [n,2,2] by a float64 eigendecomposition
    V diag(lambda^-1/2) V^T, packed (wxx, wxy, wyy)."""
    import numpy as np
    a = c.astype(np.float64)
    a = 0.5 * (a + a.transpose(0, 2, 1))
    lam, V = np.linalg.eigh(a)
    Wm = np.einsum("nij,nj,nkj->nik", V, lam ** -0.5, V)
    return np.stack([Wm[:, 0, 0], Wm[:, 0, 1], Wm[:, 1, 1]], 1)


def test_uncertainty_pnp_weights_sweep(pvb):
    """Closed-form inv(sqrtm(cov)) (cov_to_weights, csrc/common.cuh) against a float64 eigendecomposition over condition
    numbers 1..1e7, scales 1e-5..1e5 and both signs of the off-diagonal: every weight within 2 fp32 ulp (plus 1e-12 of
    the largest weight, for an off-diagonal that vanishes).  Guards: cov[0,0] < fp32(1e-6) -> zeros (fp32(1e-6) itself
    and the float above it are computed), NaN -> zeros, det <= 0 (rank 1, indefinite) -> zeros."""
    import numpy as np
    rows = []
    for kappa in (1.0, 3.0, 1e2, 1e4, 1e5, 1e6, 1e7):
        for scale in (1e-5, 1e-3, 1.0, 1e2, 1e5):
            for th in (0.0, 0.3, -0.3, 1.1, -1.1, np.pi / 2):
                R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
                rows.append(R @ np.diag([scale, scale / kappa]) @ R.T)
    c = np.asarray(rows).astype(np.float32)
    c[:, 1, 0] = c[:, 0, 1]
    got = pvb.uncertainty_pnp_weights(torch.from_numpy(c).cuda()).cpu().numpy()
    live = (c[:, 0, 0] >= np.float32(1e-6)) & (np.linalg.det(c.astype(np.float64)) > 0)
    assert live.sum() > 150 and (got[~live] == 0).all()
    want = _weights_f64(c[live])
    bar = 2 * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + 1e-12 * np.abs(want).max(1, keepdims=True)
    err = np.abs(got[live].astype(np.float64) - want)
    assert (err <= bar).all(), (np.max(err / bar), c[live][np.argmax((err / bar).max(1))])
    assert np.signbit(got[live][:, 1][np.abs(want[:, 1]) > 1e-3 * np.abs(want).max(1)]).tolist() == \
        np.signbit(want[:, 1][np.abs(want[:, 1]) > 1e-3 * np.abs(want).max(1)]).tolist()
    # the cov[0,0] guard at fp32(1e-6) and its neighbours; NaN; rank 1; indefinite; zero
    e = np.float32(1e-6)
    g = np.array([[[np.nextafter(e, np.float32(0)), 0], [0, 1]], [[e, 0], [0, 1]], [[np.nextafter(e, np.float32(1)), 0], [0, 1]],
                  [[np.nan, 0], [0, 1]], [[1, 0], [0, np.nan]], [[1, 2], [2, 4]], [[4, 2], [2, 1]], [[1, 3], [3, 1]],
                  [[1e-3, 0], [0, -1e-3]], [[0, 0], [0, 0]], [[2, 1e3], [1e3, 2]]], dtype=np.float32)
    w = pvb.uncertainty_pnp_weights(torch.from_numpy(g).cuda()).cpu().numpy()
    assert (w[0] == 0).all() and (w[3:] == 0).all()
    want = _weights_f64(g[1:3])
    assert (np.abs(w[1:3] - want) <= 2 * np.spacing(np.abs(want).astype(np.float32)) + 1e-12 * np.abs(want).max()).all()
