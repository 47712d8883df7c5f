"""GPU: the v3 chain's kernels are programmatic dependent launches (common.cuh, DESIGN.md 4): each may start while the one
before it is still running.  Bar: every result is byte-identical whether calls run back to back on one stream with no
synchronisation between them, with torch.cuda.synchronize() after each, on side streams, or from two host threads; the
pruned vote gives the keypoints and winners of the full vote (debug=True); the host-buffer entry and pvb_decode_v3 give
what the device entry gives."""
import threading

import pytest
import torch

pytestmark = pytest.mark.gpu

HN = 512


def _shape(name, B):
    from clean_pvnet_b200 import synth
    return dict(synth.CONFIGS[name], B=B)


# (shape, input seed, inlier threshold, vote seed): cfg-2, a cfg-4-shaped batch and B = 1 (not pruned: B*K < 32)
CASES = [
    (("cfg2", 16), 101, 0.99, 7),
    (("cfg4", 8), 102, 0.99, 8),
    (("cfg2", 1), 103, 0.99, 9),
    (("cfg2", 4), 104, 0.95, 10),
    (("cfg2", 16), 105, 0.999, 11),
]


@pytest.fixture(scope="module")
def inputs():
    from clean_pvnet_b200 import synth
    res = []
    for (name, B), s, t, vs in CASES:
        mask, vertex, _ = synth.make_inputs(_shape(name, B), device="cuda", seed=s)
        res.append((mask, vertex, t, vs))
    torch.cuda.synchronize()
    return res


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b))


def _calls(pvb, cases, sync):
    outs = []
    for mask, vertex, t, vs in cases:
        outs.append(pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=t, seed=vs))
        if sync:
            torch.cuda.synchronize()
    return outs


@pytest.fixture(scope="module")
def synced(pvb, inputs):
    """each call on its own: synchronised before the next starts"""
    return _calls(pvb, inputs, True)


def test_back_to_back_on_one_stream(pvb, inputs, synced):
    # twice through the list: every pair of shapes and thresholds meets at a call boundary, with no sync anywhere
    outs = _calls(pvb, inputs + inputs, False)
    torch.cuda.synchronize()
    assert _same(outs, synced + synced)


def test_side_streams(pvb, inputs, synced):
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = []
    for i, case in enumerate(inputs + inputs):
        with torch.cuda.stream(streams[i % 2]):
            outs += _calls(pvb, [case], False)
    torch.cuda.synchronize()
    assert _same(outs, synced + synced)


def test_two_host_threads(pvb, inputs, synced):
    # each thread its own stream and its own cases (the cases differ in shape or threshold, so no call descriptor is shared)
    parts = [[0, 2], [1, 3, 4]]
    res, errs = [None, None], []

    def work(j):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                cases = [inputs[i] for i in parts[j]]
                res[j] = _calls(pvb, cases + cases, False)
            s.synchronize()
        except Exception as e:  # pragma: no cover - reported below
            errs.append(e)

    th = [threading.Thread(target=work, args=(j,)) for j in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for j in range(2):
        want = [synced[i] for i in parts[j]]
        assert _same(res[j], want + want)


def _win_of_last_call(mask, vertex, t, vs):
    """the winners the last (pruned) call on the current stream left in its workspace, cloned in stream order"""
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    lib = _lib.load()
    m, v = rv._check_inputs(mask, vertex)
    d = rv._make_desc(m, v, HN, t, 5, 30000, _lib.PVB_SELECT_BYTE, vs, 0, None)
    ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
    L = _lib.PvbLayout()
    _lib.check(lib.pvb_workspace_layout(d, L))
    B, K = d.B, d.K
    return ws[L.win:L.win + B * K * 8].view(torch.float32).view(B, K, 2).clone()


def test_pruned_equals_full_vote(pvb, inputs):
    got = []
    for mask, vertex, t, vs in inputs:
        out = pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=t, seed=vs)
        win = _win_of_last_call(mask, vertex, t, vs)
        full, dbg = pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=t, seed=vs, debug=True)
        got.append((out, win, full, dbg["win"]))
    torch.cuda.synchronize()
    for out, win, full, fwin in got:
        assert torch.equal(_bits(out), _bits(full))
        assert torch.equal(_bits(win), _bits(fwin))


def test_host_buffer_entry(pvb, inputs, synced):
    # chunks of 4 images are pruned (B*K = 36), chunks of 1 are not
    for chunk in (4, 1):
        outs = []
        for mask, vertex, t, vs in inputs[:4]:
            outs.append(pvb.ransac_voting_layer_v3_host(mask.cpu().pin_memory(), vertex.cpu().pin_memory(), HN,
                                                        inlier_thresh=t, seed=vs, chunk_images=chunk))
        assert _same(outs, [o.cpu() for o in synced[:4]])


def test_decode_v3_back_to_back(pvb):
    from clean_pvnet_b200 import synth
    nets = []
    for (name, B), s in ((("cfg2", 4), 111), (("cfg2", 1), 112), (("cfg4", 2), 113)):
        mask, vertex, _ = synth.make_inputs(_shape(name, B), device="cuda", seed=s, layout="planar")
        Bn, H, W, K, _ = vertex.shape
        g = torch.Generator(device="cuda").manual_seed(s)
        seg = torch.randn((Bn, 2, H, W), generator=g, device="cuda") * 0.3
        seg[:, 1] += (mask.float() * 2 - 1) * 1.5
        nets.append({"seg": seg, "vertex": vertex.permute(0, 3, 4, 1, 2).reshape(Bn, 2 * K, H, W).contiguous()})
    torch.cuda.synchronize()

    def run(fused, sync):
        res = []
        for i, net in enumerate(nets + nets):
            o = pvb.decode_keypoint(dict(net), un_pnp=False, seed=40 + i % len(nets), fused=fused)
            res += [o["mask"], o["kpt_2d"]]
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return res

    want = run(False, True)
    assert _same(run(True, False), want)
    assert _same(run(True, True), want)
