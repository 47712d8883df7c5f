"""GPU tests of the CenterNet decode (DESIGN.md 8j): decode_detections against the reference's own decode
(tests/golden/ct_decode.npz) and against the restatement run on CUDA torch on seeded cases with ties and NaN.  CUDA
torch's topk does not order equal values by a fixed rule, so the decode orders them by class and pixel index: every row
equals a stable-sort restatement bit for bit, and the two-topk restatement row for row where scores are unique, with
tied rows compared as sets; batches, channels-last and sliced inputs, batch independence, determinism, sync-free
execution on a side stream, CUDA-graph capture; detection_boxes against get_affine_transform / affine_transform; the
batched chain against the cascade's crop; and the patched decode_detection."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import crop_cases as cc
import ct_decode_cases as dc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ct_decode.npz")


def _bits(t):
    """float32 bits with every NaN as one pattern, so NaN rows compare equal and -0 differs from +0."""
    t = t.detach().float().cpu().contiguous()
    t = torch.where(t.isnan(), torch.full_like(t, float("nan")), t)
    return t.view(torch.int32)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _restated(lg, wh, K, clip=True):
    return dc.restate_decode_ordered(lg, wh, K, clip)


def _check_against_topk(det, ct, want_det, want_ct, name):
    """det / ct against CUDA torch's two-topk decode: the score column bit for bit; a row whose score no other row of
    the image shares, bit for bit; a group of tied rows as a set, except the group the K-th row ends in, whose members
    torch picks by its own order (the stable-sort comparison pins ours)."""
    rows, want_rows = torch.cat([det, ct], -1), torch.cat([want_det, want_ct], -1)
    assert torch.equal(_bits(det[..., 4]), _bits(want_det[..., 4])), name
    for b in range(det.shape[0]):
        sc = _bits(det[b, :, 4])
        last = sc[-1]
        for v in sc.unique():
            if v == last:
                continue
            sel = (sc == v).nonzero()[:, 0]
            got = sorted(map(tuple, _bits(rows[b, sel]).tolist()))
            want = sorted(map(tuple, _bits(want_rows[b, sel]).tolist()))
            assert got == want, (name, b, int(v), sel.tolist())


def test_cuda_topk_tie_order_is_not_a_fixed_rule():
    """What the decode's tie order rests on, as measured: NaN ranks above +inf, and on a long slice equal values come
    out in ascending index; on a short slice (the second topk over C*K values, or K close to its length) they do not."""
    for n in (25024, 3000):
        x = torch.zeros(n, device="cuda")
        x[n // 3] = x[n // 2] = 1.0
        v, i = torch.topk(x, 100)
        assert i[:2].tolist() == [n // 3, n // 2]
        assert i[2:].tolist() == [j for j in range(n) if j not in (n // 3, n // 2)][:98], n
        x[5] = float("inf")
        x[n - 1] = float("nan")
        v, i = torch.topk(x, 3)
        assert i.tolist() == [n - 1, 5, n // 3]
    lg = torch.from_numpy(next(c for c in dc.cases() if c[0] == "borders")[1]).cuda()
    heat = dc._peaks(lg).reshape(1, -1)
    _, i = torch.topk(heat, 20)
    print("CUDA torch topk order of 12 tied zeros after 8 peaks:", i[0, 8:].tolist())


def test_cuda_max_pool_lets_nan_win():
    heat = torch.tensor([[[[0.5, 0.1, 0.2, 0.3], [0.1, float("nan"), 0.1, 0.9], [0.2, 0.1, 0.1, 0.1]]]], device="cuda")
    hmax = torch.nn.functional.max_pool2d(heat, 3, stride=1, padding=1)
    kept = heat * (hmax == heat).float()
    assert kept[0, 0, 1, 1].isnan() and kept[0, 0, 0, 0] == 0 and kept[0, 0, 2, 2] == 0
    assert kept[0, 0, 1, 3] == heat[0, 0, 1, 3]              # its window (columns 2-3) does not reach the NaN
    assert int(kept.isnan().sum()) == 1 and int((kept != 0).sum()) == 2


def test_decode_equals_the_reference_golden(pvb):
    g = np.load(GOLDEN)
    for c, name in enumerate(g["names"]):
        lg, wh = torch.from_numpy(g[f"logits{c}"]).cuda(), torch.from_numpy(g[f"wh{c}"]).cuda()
        K = int(g[f"K{c}"])
        ct, det = pvb.decode_detections(lg, wh, K)
        want = torch.from_numpy(g[f"detection{c}"])
        # the fixture comes from CPU torch, whose sigmoid differs from CUDA torch's in the last bits: everything but
        # the score is equal, the score is CUDA torch's (the restatement on the device), 2 ulp at most from CPU's
        assert torch.equal(ct.cpu(), torch.from_numpy(g[f"ct{c}"])), name
        assert torch.equal(det.cpu()[..., [0, 1, 2, 3, 5]], want[..., [0, 1, 2, 3, 5]]), name
        assert torch.equal(det, _restated(lg, wh, K)[1]) and torch.equal(det, dc.restate_decode(lg, wh, K)[1]), name
        ulp = torch.abs(det.cpu()[..., 4].view(torch.int32) - want[..., 4].view(torch.int32))
        assert int(ulp.max()) <= 2, name


@pytest.mark.parametrize("case", [c[0] for c in dc.cases()])
def test_decode_equals_cuda_torch(pvb, case):
    name, lg, wh, K = next(c for c in dc.cases() if c[0] == case)
    lg, wh = torch.from_numpy(lg).cuda(), torch.from_numpy(wh).cuda()
    for clip in (True, False):
        want_ct, want_det = _restated(lg, wh, K, clip)
        ct, det = pvb.decode_detections(lg, wh, K, clip)
        assert _same(ct, want_ct), (name, clip)
        bad = (_bits(det) != _bits(want_det)).any(-1).nonzero()
        assert bad.numel() == 0, (name, clip, bad[:8].tolist())
        _check_against_topk(det, ct, *reversed(dc.restate_decode(lg, wh, K, clip)), (name, clip))


@pytest.mark.parametrize("B,C,hw", [(1, 1, dc.TEST_HW), (4, 30, dc.TEST_HW), (32, 1, dc.TRAIN_HW),
                                    (32, 30, dc.TRAIN_HW), (4, 30, (512, 384))])
def test_batches_layouts_and_independence(pvb, B, C, hw):
    rng = np.random.default_rng(B * 100 + C)
    lg = torch.from_numpy(dc.blobs(rng, B, C, *hw, noise=0.3)).cuda()
    wh = torch.from_numpy(dc._wh(rng, B, *hw)).cuda()
    want = _restated(lg, wh, 100)
    got = pvb.decode_detections(lg, wh)
    assert _same(got[0], want[0]) and _same(got[1], want[1])
    _check_against_topk(got[1], got[0], *reversed(dc.restate_decode(lg, wh, 100)), (B, C, hw))
    # channels-last logits, and both maps sliced out of wider buffers
    cl = lg.contiguous(memory_format=torch.channels_last)
    big = torch.full((B, C + 2, hw[0] + 3, hw[1] + 5), float("nan"), device="cuda")
    big[:, 1:C + 1, 2:hw[0] + 2, 1:hw[1] + 1] = lg
    sl = big[:, 1:C + 1, 2:hw[0] + 2, 1:hw[1] + 1]
    bigw = torch.full((B, 4, hw[0], hw[1] + 7), float("nan"), device="cuda")
    bigw[:, 1:3, :, 3:hw[1] + 3] = wh
    slw = bigw[:, 1:3, :, 3:hw[1] + 3]
    for l2, w2 in ((cl, wh), (sl, slw), (cl, slw)):
        got2 = pvb.decode_detections(l2, w2)
        assert _same(got2[0], got[0]) and _same(got2[1], got[1])
    # determinism, and an image alone equals the same image in the batch
    again = pvb.decode_detections(lg, wh)
    assert _same(again[0], got[0]) and _same(again[1], got[1])
    for b in {0, B - 1, B // 2}:
        one = pvb.decode_detections(lg[b:b + 1], wh[b:b + 1])
        assert _same(one[0][0], got[0][b]) and _same(one[1][0], got[1][b]), b


def test_no_host_sync_side_stream_and_graph(pvb):
    rng = np.random.default_rng(7)
    lg = torch.from_numpy(dc.blobs(rng, 4, 30, *dc.TRAIN_HW, noise=0.3)).cuda()
    wh = torch.from_numpy(dc._wh(rng, 4, *dc.TRAIN_HW)).cuda()
    want = pvb.decode_detections(lg, wh)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.stream(side):
            got = pvb.decode_detections(lg, wh)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.current_stream().wait_stream(side)
    assert _same(got[0], want[0]) and _same(got[1], want[1])

    static_lg, static_wh = lg.clone(), wh.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pvb.decode_detections(static_lg, static_wh)            # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = pvb.decode_detections(static_lg, static_wh)
    lg2 = torch.from_numpy(dc.blobs(rng, 4, 30, *dc.TRAIN_HW, noise=0.3)).cuda()
    static_lg.copy_(lg2)
    graph.replay()
    torch.cuda.synchronize()
    want2 = _restated(lg2, wh, 100)
    assert _same(out[0], want2[0]) and _same(out[1], want2[1])


def _np_boxes(det, center, scale, w, h, down_ratio=4):
    """The consumers' host loop with get_affine_transform / affine_transform restated (crop_cases)."""
    out = []
    for b in range(det.shape[0]):
        Minv = cc.crop_matrices(np.asarray(center[b], np.float32), np.float32(scale[b]), w, h)[1]
        box = det[b, :, :4] * np.float32(down_ratio)
        out.append(np.stack([cc.dot_affine(bx.reshape(-1, 2), Minv).ravel() for bx in box]))
    return np.stack(out)


def test_detection_boxes(pvb):
    g = np.load(GOLDEN)
    w, h = dc.BOX_INPUT_SIZE
    for c, name in enumerate(g["names"]):
        det = torch.from_numpy(g[f"detection{c}"]).cuda()
        B = det.shape[0]
        center = np.tile(np.array(dc.BOX_CENTER, np.float32), (B, 1))
        scale = np.tile(np.array(dc.BOX_SCALE, np.float64), (B, 1))
        got = pvb.detection_boxes(det, center, scale, (w, h)).cpu().numpy()
        assert np.abs(got - g[f"boxes{c}"]).max() <= 1e-12, name
        got1 = pvb.detection_boxes(det, torch.from_numpy(center), torch.from_numpy(scale[:, 0]), (w, h))
        assert np.array_equal(got1.cpu().numpy(), got)
    rng = np.random.default_rng(9)
    det = torch.from_numpy(rng.uniform(-20, 200, (8, 100, 6)).astype(np.float32)).cuda()
    center = rng.uniform(200, 500, (8, 2)).astype(np.float32)
    scale = rng.integers(400, 1000, 8).astype(np.float64)
    got = pvb.detection_boxes(det, center, scale, (512, 416)).cpu().numpy()
    assert np.abs(got - _np_boxes(det.cpu().numpy(), center, scale, 512, 416)).max() <= 1e-12


def test_batched_chain_equals_cascade_crop(pvb, monkeypatch):
    """decode_detections -> detection_boxes[:, :1] -> crop_device with the cascade's arguments, with its ct_score = 0
    cut on the device, equals cascade_crop's output['inp'] image by image for a batch of 4."""
    du = types.SimpleNamespace(get_affine_transform=lambda c, s, rot, size, inv=0: cc.crop_matrices(
        c, np.float32(s[0] if np.ndim(s) else s), *size)[inv], affine_transform=cc.dot_affine)
    tc = types.SimpleNamespace(scale_ratio=2.4, mean=cc.MEAN.reshape(1, 1, 3), std=cc.STD.reshape(1, 1, 3))
    res = types.ModuleType("lib.networks.ct_pvnet.res")
    res.data_utils, res.tless_config = du, tc
    res.tless_pvnet_utils = types.SimpleNamespace(input_scale=np.array([256, 256]))
    monkeypatch.setitem(sys.modules, "lib.networks.ct_pvnet.res", res)
    rng = np.random.default_rng(21)
    B = 4
    imgs = torch.from_numpy(cc.random_images(rng, B)).cuda()
    lg = torch.from_numpy(dc.blobs(rng, B, 30, *dc.TEST_HW, noise=0.3)).cuda()
    lg[3] = float("-inf")                          # image 3: every score is 0, so the ct_score = 0 cut drops its box
    wh = torch.from_numpy(dc._wh(rng, B, *dc.TEST_HW)).cuda()
    meta_c = np.tile(np.array([360.0, 270.0], np.float32), (B, 1))
    meta_s = np.tile(np.array([720.0, 720.0], np.float32), (B, 1))
    ct, det = pvb.decode_detections(lg, wh)
    boxes = pvb.detection_boxes(det, meta_c, meta_s, (736, 544))[:, :1]
    keep = det[:, 0, 4] > 0
    idx = keep.nonzero()[:, 0]
    inp = pvb.crop.crop_device(imgs, boxes[idx, 0], idx, (256, 256), 2.4, 0.0, False, True, False,
                               cc.MEAN.reshape(3), cc.STD.reshape(3))[0]
    row = torch.cumsum(keep.int(), 0) - 1
    for b in range(B):
        batch = {'meta': {'center': torch.from_numpy(meta_c[b:b + 1]), 'scale': torch.from_numpy(meta_s[b:b + 1])},
                 'inp': torch.zeros((1, 3, 544, 736))}
        output = {'detection': det[b:b + 1]}
        want = pvb.crop.cascade_crop(imgs[b:b + 1], None, batch, output)
        if bool(keep[b]):
            assert torch.equal(inp[int(row[b])], want[0]), b
        else:
            assert want == [], b


def test_patched_decode_detection(pvb, monkeypatch):
    """install_ct_decode_as_reference on a stand-in lib.networks.ct.dla: the patched Network.decode_detection writes
    output['ct'] / output['detection'] equal to the restated reference and returns them."""
    for name in ("lib", "lib.networks", "lib.networks.ct"):
        mod = types.ModuleType(name)
        mod.__path__ = []
        monkeypatch.setitem(sys.modules, name, mod)
    dla = types.ModuleType("lib.networks.ct.dla")

    class Network:
        def decode_detection(self, output, h, w):
            raise AssertionError("not patched")

    dla.Network = Network
    monkeypatch.setitem(sys.modules, "lib.networks.ct.dla", dla)
    monkeypatch.setattr(sys.modules["lib.networks.ct"], "dla", dla, raising=False)
    pvb.install_ct_decode_as_reference()
    pvb.install_ct_decode_as_reference()
    rng = np.random.default_rng(5)
    lg = torch.from_numpy(dc.blobs(rng, 2, 30, *dc.TEST_HW, noise=0.3)).cuda()
    wh = torch.from_numpy(dc._wh(rng, 2, *dc.TEST_HW)).cuda()
    output = {'ct_hm': lg, 'wh': wh}
    ct, det = Network().decode_detection(output, *dc.TEST_HW)
    want = _restated(lg, wh, 100)
    assert output['ct'] is ct and output['detection'] is det
    assert _same(ct, want[0]) and _same(det, want[1])
