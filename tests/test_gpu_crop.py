"""GPU tests of T-LESS's PVNet crop (DESIGN.md 8g): crop_inputs against the reference's own pvnet_transform outputs
(tests/golden/tless_crop.npz) and against cv2.warpAffine + numpy on fresh seeded cases, the device crop matrices against
cv2.getAffineTransform, uncrop_keypoints against the golden file, batch independence and determinism, sync-free
execution on a side stream, uncrop -> pnp_batch against affine_transform + cv2.solvePnP, the patched cascade crop, and
warp_affine_batch against cv2."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import crop_cases as cc
from pnp_iter_cases import rel_diff

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "tless_crop.npz")
K_TLESS = np.array([[1075.65091572, 0.0, 367.06888344], [0.0, 1073.90347929, 247.72159802], [0.0, 0.0, 1.0]])


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float64)).view(np.uint64)


def _cv2_crop(img, box, size, scale_ratio, box_ratio, mask=True):
    """pvnet_transform with cv2 itself doing the matrix and the warp: (inp [3,h,w], u8 [h,w,3], M, Minv)."""
    w, h = size
    c, s = cc.center_scale(box, scale_ratio)
    src, dst = cc.crop_points(c, s, w, h)
    M, Minv = cv2.getAffineTransform(src, dst), cv2.getAffineTransform(dst, src)
    u8 = cv2.warpAffine(img, M, (w, h), flags=cv2.INTER_LINEAR)
    if mask:
        x0, y0, x1, y1 = cc.magnify(box, M, box_ratio, w, h)
        keep = np.zeros_like(u8)
        keep[y0:y1 + 1, x0:x1 + 1] = u8[y0:y1 + 1, x0:x1 + 1]
        u8 = keep
    return cc.normalise(u8), u8, M, Minv


def test_crop_inputs_equals_the_reference_golden(pvb):
    print("cv2", cv2.__version__)
    g = np.load(GOLDEN)
    img = torch.from_numpy(cc.pattern_images(g["img_params"])).cuda()
    for name in cc.CONFIGS:
        w, h, scale_ratio, box_ratio = g[f"{name}_config"]
        inp, center, scale, u8 = pvb.crop_inputs(img, g[f"{name}_boxes"], g[f"{name}_index"], (int(w), int(h)),
                                                 float(scale_ratio), float(box_ratio), return_uint8=True)
        inp, u8 = inp.cpu().numpy(), u8.cpu().numpy()
        assert np.array_equal(u8, g[f"{name}_crop"]), name
        assert [cc.sha256(x) for x in inp] == list(g[f"{name}_inp_sha256"]), name
        assert np.array_equal(center.cpu().numpy(), g[f"{name}_center"])
        assert np.array_equal(scale.cpu().numpy(), g[f"{name}_scale"].astype(np.float32))


@pytest.mark.parametrize("n,contiguous", [(1, True), (16, False), (1024, True), (1024, False)])
def test_crop_inputs_equals_cv2_on_fresh_cases(pvb, n, contiguous):
    rng = np.random.default_rng(100 + n + int(contiguous))
    imgs = cc.random_images(rng, 3)
    boxes = np.concatenate([cc.random_boxes(rng, n - 1), cc.DEGENERATE[:1]]) if n > 1 else cc.random_boxes(rng, 1)
    index = rng.integers(0, 3, n)
    size, scale_ratio, box_ratio = ((128, 128), 1.2, 1.1) if n > 16 else ((256, 256), 2.4, 1.2)
    if contiguous:
        dev_img = torch.from_numpy(imgs).cuda()
    else:                                                   # channels strided inside a 4-channel buffer, rows padded
        buf = torch.zeros((3, 540, 736, 4), dtype=torch.uint8, device="cuda")
        buf[:, :, :720, :3] = torch.from_numpy(imgs).cuda()
        dev_img = buf[:, :, :720, :3]
        assert not dev_img.is_contiguous()
    inp, center, scale, u8 = pvb.crop_inputs(dev_img, boxes, index, size, scale_ratio, box_ratio, return_uint8=True)
    inp_h, u8_h = inp.cpu().numpy(), u8.cpu().numpy()
    for i in range(n):
        want_inp, want_u8, _, _ = _cv2_crop(imgs[index[i]], boxes[i], size, scale_ratio, box_ratio)
        assert np.array_equal(u8_h[i], want_u8), i
        assert np.array_equal(inp_h[i].view(np.uint32), want_inp.view(np.uint32)), i


def test_device_matrices_equal_get_affine_transform(pvb):
    rng = np.random.default_rng(11)
    boxes = np.concatenate([cc.random_boxes(rng, 3000), cc.DEGENERATE])
    img = torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device="cuda")
    for size, center_f64 in (((256, 256), False), ((128, 96), True)):
        _, _, c, s, M, Minv = pvb.crop.crop_device(img, boxes, None, size, 2.4, 1.2, True, center_f64)
        c, s, M, Minv = c.cpu().numpy(), s.cpu().numpy(), M.cpu().numpy(), Minv.cpu().numpy()
        for i, b in enumerate(boxes):
            cw, sw = cc.center_scale(b, 2.4, center_f32=not center_f64)
            assert np.array_equal(_bits(c[i]), _bits(cw)) and s[i] == sw, i
            src, dst = cc.crop_points(cw, sw, *size)
            assert np.array_equal(_bits(M[i]), _bits(cv2.getAffineTransform(src, dst))), i
            assert np.array_equal(_bits(Minv[i]), _bits(cv2.getAffineTransform(dst, src))), i


def test_uncrop_keypoints_matches_the_golden(pvb):
    g = np.load(GOLDEN)
    for name in cc.CONFIGS:
        w, h = (int(v) for v in g[f"{name}_config"][:2])
        out = pvb.uncrop_keypoints(torch.from_numpy(g[f"{name}_kpt"]).cuda(), g[f"{name}_center"], g[f"{name}_scale"],
                                   (w, h)).cpu().numpy()
        assert np.abs(out - g[f"{name}_uncrop"]).max() <= 1e-12, name
        f32 = pvb.uncrop_keypoints(torch.from_numpy(g[f"{name}_kpt"]).cuda(), g[f"{name}_center"],
                                   g[f"{name}_scale"].astype(np.float32), (w, h)).cpu().numpy()
        assert np.array_equal(out, f32)           # scale is rounded to float32 either way, as get_affine_transform does


def test_batch_independence_and_determinism(pvb):
    rng = np.random.default_rng(12)
    imgs = torch.from_numpy(cc.random_images(rng, 2)).cuda()
    boxes = cc.random_boxes(rng, 1024)
    index = rng.integers(0, 2, 1024)
    a = pvb.crop_inputs(imgs, boxes, index, return_uint8=True)
    b = pvb.crop_inputs(imgs, boxes, index, return_uint8=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    for i in (0, 517, 1023):
        one = pvb.crop_inputs(imgs, boxes[i:i + 1], index[i:i + 1], return_uint8=True)
        for x, y in zip(one, a):
            assert torch.equal(x[0], y[i]), i


def test_no_host_sync_and_side_stream(pvb):
    rng = np.random.default_rng(13)
    imgs = torch.from_numpy(cc.random_images(rng, 2)).cuda()
    boxes = torch.from_numpy(cc.random_boxes(rng, 64)).cuda()
    index = torch.from_numpy(rng.integers(0, 2, 64)).cuda()
    kpt = torch.rand((64, 9, 2), device="cuda") * 256
    M = torch.from_numpy(np.stack([cc.crop_matrices(*cc.center_scale(b, 2.4), 256, 256)[0] for b in
                                   boxes.cpu().numpy()])).cuda()
    want = pvb.crop_inputs(imgs, boxes, index)
    want_un = pvb.uncrop_keypoints(kpt, want[1], want[2])
    want_w = pvb.warp_affine_batch(imgs, M, (256, 256), index)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.stream(side):
            got = pvb.crop_inputs(imgs, boxes, index)
            got_un = pvb.uncrop_keypoints(kpt, got[1], got[2])
            got_w = pvb.warp_affine_batch(imgs, M, (256, 256), index)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.current_stream().wait_stream(side)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert torch.equal(got_un, want_un) and torch.equal(got_w, want_w)


def test_uncrop_then_pnp_batch_matches_affine_transform_and_solvepnp(pvb):
    """Crop-frame keypoints of posed models -> uncrop_keypoints -> pnp_batch, against a per-box loop of the reference's
    affine_transform + cv2.solvePnP(ITERATIVE), at the pnp_batch pin's bar (1e-8)."""
    rng = np.random.default_rng(14)
    n, K = 32, 9
    model = rng.uniform(-40, 40, (K, 3))
    kpt_crop, centers, scales, want = [], [], [], []
    for i in range(n):
        R = cv2.Rodrigues(rng.uniform(-1, 1, 3))[0]
        t = np.array([rng.uniform(-100, 100), rng.uniform(-80, 80), rng.uniform(500, 900)])
        uv = (model @ R.T + t) @ K_TLESS.T
        uv = uv[:, :2] / uv[:, 2:]
        box = [uv[:, 0].min() - 5, uv[:, 1].min() - 5, uv[:, 0].max() + 5, uv[:, 1].max() + 5]
        c, s = cc.center_scale(box, 2.4)
        M, Minv = cc.crop_matrices(c, s, 256, 256)
        k = (cc.dot_affine(uv, M) + rng.normal(0, 0.5, (K, 2))).astype(np.float32)   # the network's crop-frame output
        pts = cc.dot_affine(k, Minv)
        ok, rvec, tvec = cv2.solvePnP(model, pts.reshape(-1, 1, 2), K_TLESS, None, flags=cv2.SOLVEPNP_ITERATIVE)
        want.append(np.hstack([cv2.Rodrigues(rvec)[0], tvec.reshape(3, 1)]))
        kpt_crop.append(k); centers.append(c.astype(np.float32)); scales.append(np.float32(s))
    pts2d = pvb.uncrop_keypoints(torch.from_numpy(np.stack(kpt_crop)).cuda(), np.stack(centers), np.array(scales))
    pose = pvb.pnp_batch(model, pts2d, K_TLESS).cpu().numpy()
    for i in range(n):
        assert rel_diff(want[i], pose[i]) <= 1e-8, i


def test_patched_cascade_crop_matches_the_restated_reference(pvb, monkeypatch):
    """res.crop with its module's data_utils / tless_config / tless_pvnet_utils; the image and the detection are CUDA
    tensors.  The expected result is res._crop's code path restated on the host: the box through trans_output_inv, a
    float64 centre, no box mask."""
    du = types.SimpleNamespace(get_affine_transform=lambda c, s, rot, size, inv=0: cc.crop_matrices(
        c, np.float32(s[0] if np.ndim(s) else s), *size)[inv], affine_transform=cc.dot_affine)
    tc = types.SimpleNamespace(scale_ratio=2.4, mean=cc.MEAN.reshape(1, 1, 3), std=cc.STD.reshape(1, 1, 3))
    res = types.ModuleType("lib.networks.ct_pvnet.res")
    res.data_utils, res.tless_config = du, tc
    res.tless_pvnet_utils = types.SimpleNamespace(input_scale=np.array([256, 256]))
    monkeypatch.setitem(sys.modules, "lib.networks.ct_pvnet.res", res)
    rng = np.random.default_rng(15)
    img = cc.random_images(rng, 1)
    det = torch.tensor([[[30.5, 20.25, 70.75, 61.0, 0.9, 3.0]]], device="cuda")
    meta_c, meta_s = np.array([360.0, 270.0], np.float32), np.array([720.0, 720.0], np.float32)
    batch = {'meta': {'center': torch.from_numpy(meta_c[None]), 'scale': torch.from_numpy(meta_s[None])},
             'inp': torch.zeros((1, 3, 544, 736))}
    output = {'detection': det}
    inp = pvb.crop.cascade_crop(torch.from_numpy(img).cuda(), det, batch, output)
    trans_output_inv = cc.crop_matrices(meta_c, meta_s[0], 736, 544)[1]
    box = cc.dot_affine(det[0, 0, :4].cpu().numpy().reshape(-1, 2) * 4, trans_output_inv).ravel()
    want_inp, _, c, s, _, _ = cc.crop_restated(img[0], box, (256, 256), 2.4, 1.2, mask_to_box=False, center_f32=False)
    assert output['inp'] is inp and inp.is_cuda and inp.shape == (1, 3, 256, 256)
    assert np.array_equal(inp[0].cpu().numpy().view(np.uint32), want_inp.view(np.uint32))
    assert isinstance(output['center'], tuple) and np.array_equal(output['center'][0], c)
    assert isinstance(output['scale'], tuple) and output['scale'][0] == s
    output2 = {'detection': torch.tensor([[[30.5, 20.25, 70.75, 61.0, -1.0, 3.0]]], device="cuda")}
    assert pvb.crop.cascade_crop(torch.from_numpy(img).cuda(), None, batch, output2) == [] and output2['inp'] == []


def test_warp_affine_batch_equals_cv2(pvb):
    """The detector's full-image resize (tless_test_utils.augment: 720x540 -> 736x544), crops from several images, and
    one- and four-channel images."""
    rng = np.random.default_rng(16)
    imgs = cc.random_images(rng, 2)
    src, dst = cc.crop_points(np.array([360.0, 270.0], np.float32), 720.0, 736, 544)
    M = cv2.getAffineTransform(src, dst)
    out = pvb.warp_affine_batch(torch.from_numpy(imgs).cuda(), np.stack([M, M]), (736, 544), [0, 1]).cpu().numpy()
    for i in range(2):
        assert np.array_equal(out[i], cv2.warpAffine(imgs[i], M, (736, 544), flags=cv2.INTER_LINEAR))
    boxes = cc.random_boxes(rng, 24)
    Ms = np.stack([cc.crop_matrices(*cc.center_scale(b, 1.5), 200, 150)[0] for b in boxes])
    idx = rng.integers(0, 2, 24)
    out = pvb.warp_affine_batch(torch.from_numpy(imgs).cuda(), Ms, (200, 150), idx).cpu().numpy()
    for i in range(24):
        assert np.array_equal(out[i], cv2.warpAffine(imgs[idx[i]], Ms[i], (200, 150), flags=cv2.INTER_LINEAR)), i
    g = np.ascontiguousarray(imgs[0, :, :, 2])
    og = pvb.warp_affine_batch(torch.from_numpy(g).cuda(), Ms[0], (200, 150)).cpu().numpy()
    assert og.shape == (1, 150, 200) and np.array_equal(og[0], cv2.warpAffine(g, Ms[0], (200, 150), flags=cv2.INTER_LINEAR))
    four = np.concatenate([imgs[1], imgs[0][:, :, :1]], axis=2)
    o4 = pvb.warp_affine_batch(torch.from_numpy(four).cuda(), Ms[1], (200, 150)).cpu().numpy()
    assert np.array_equal(o4[0], cv2.warpAffine(four, Ms[1], (200, 150), flags=cv2.INTER_LINEAR))
