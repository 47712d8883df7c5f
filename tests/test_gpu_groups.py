"""Grouped launch of the pruned v3 entries (DESIGN.md 4.4): a call whose every group still prunes runs as groups of
consecutive images on internal streams.  A grouped call must write the same bytes as the same call forced into one chain
(pvb_set_group_tuning(1, 0)): the keypoints, and the whole workspace -- header, bitmaps, pixels, directions, hypotheses,
counts, refit partials and the prune regions -- which is zero-filled before each compared call so that bytes a call does
not write compare equal too."""
import contextlib
import json
import threading

import pytest
import torch

from clean_pvnet_b200 import _lib, decode, ransac_voting_gpu as rv, synth

pytestmark = pytest.mark.gpu

HN = 512


def _shape(B, K, H=240, W=320):
    return dict(B=B, H=H, W=W, K=K, hn=HN, fill=(0.25, 0.35), kind="blob")


@contextlib.contextmanager
def _groups(n):
    lib = _lib.load()
    _lib.check(lib.pvb_set_group_tuning(n, 0))
    try:
        yield
    finally:
        _lib.check(lib.pvb_set_group_tuning(0, 0))


def _ws():
    return rv._workspaces[(torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)]


def _call(pvb, mask, vertex, thresh, seed, groups):
    """(keypoints, workspace bytes) of one call on the current stream, the workspace zero-filled before it."""
    with _groups(groups):
        pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=thresh, seed=seed)      # sizes the workspace
        ws = _ws()
        ws.zero_()
        out = pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=thresh, seed=seed)
        torch.cuda.synchronize()
        return out.clone(), ws.clone()


def _grouped(pvb, mask, vertex, tmp_path):
    """True when the default call ran as groups: its kernels then ran on more than one stream."""
    pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=0.99, seed=5)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        pvb.ransac_voting_layer_v3(mask, vertex, HN, inlier_thresh=0.99, seed=5)
        torch.cuda.synchronize()
    path = str(tmp_path / "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as fh:
        streams = {e["tid"] for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel"}
    assert streams
    return len(streams) > 1


def _assert_same(a, b):
    assert torch.equal(a[0], b[0]), "keypoints differ"
    diff = (a[1] != b[1]).nonzero()
    assert diff.numel() == 0, f"{diff.numel()} workspace bytes differ, first at byte {int(diff[0])}"


@pytest.mark.parametrize("cfg,B,thresh", [
    ("cfg2", None, 0.99), ("cfg2", None, 0.95), ("cfg2", None, 0.9),
    ("cfg4", 32, 0.99),
    (_shape(13, 9), None, 0.99),            # uneven: groups of 6 and 7 images
])
def test_grouped_call_writes_the_one_group_bytes(pvb, tmp_path, cfg, B, thresh):
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=41, B=B)
    assert _grouped(pvb, mask, vertex, tmp_path)
    _assert_same(_call(pvb, mask, vertex, thresh, 7, 0), _call(pvb, mask, vertex, thresh, 7, 1))


@pytest.mark.parametrize("B,K,split", [(8, 8, True), (7, 8, False), (4, 9, False)])
def test_split_only_where_every_group_prunes(pvb, tmp_path, B, K, split):
    """2 groups of 4 x 8 = 32 (image, keypoint) pairs pass the prune gate; 7 images of 8 keypoints would leave a group
    of 3 x 8 = 24 and run as one chain; 4 x 9 = 36 pairs prune, but 2 x 9 would not."""
    mask, vertex, _ = synth.make_inputs(_shape(B, K), device="cuda", seed=43)
    assert _grouped(pvb, mask, vertex, tmp_path) == split
    _assert_same(_call(pvb, mask, vertex, 0.99, 8, 0), _call(pvb, mask, vertex, 0.99, 8, 1))


def _batches(n, seed):
    return [synth.make_inputs("cfg2", device="cuda", seed=seed + i)[:2] for i in range(n)]


def _one_group(pvb, batches, seed0):
    with _groups(1):
        outs = [pvb.ransac_voting_layer_v3(m, v, HN, inlier_thresh=0.99, seed=seed0 + i) for i, (m, v) in enumerate(batches)]
        torch.cuda.synchronize()
    return outs


def test_back_to_back_calls_on_one_stream(pvb):
    """Consecutive calls share the workspace; the next call's header memset follows the previous call's join."""
    batches = _batches(4, 50)
    want = _one_group(pvb, batches, 100)
    got = [pvb.ransac_voting_layer_v3(m, v, HN, inlier_thresh=0.99, seed=100 + i) for i, (m, v) in enumerate(batches)]
    torch.cuda.synchronize()
    for g, w in zip(got, want):
        assert torch.equal(g, w)


def test_two_caller_streams_from_one_thread(pvb):
    batches = _batches(4, 60)
    want = _one_group(pvb, batches, 200)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    got = []
    for i, (m, v) in enumerate(batches):
        with torch.cuda.stream(streams[i % 2]):
            got.append(pvb.ransac_voting_layer_v3(m, v, HN, inlier_thresh=0.99, seed=200 + i))
    for s in streams:
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for g, w in zip(got, want):
        assert torch.equal(g, w)


def test_two_host_threads(pvb):
    # one seed for every call: the Python layer shares one cached descriptor per shape between threads
    batches = _batches(2, 70)
    with _groups(1):
        want = [pvb.ransac_voting_layer_v3(m, v, HN, inlier_thresh=0.99, seed=300) for m, v in batches]
        torch.cuda.synchronize()
    got, errors = {}, []

    def work(t):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for r in range(3):
                    m, v = batches[t]
                    got[(t, r)] = pvb.ransac_voting_layer_v3(m, v, HN, inlier_thresh=0.99, seed=300)
            s.synchronize()
        except Exception as e:          # reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for (t, r), out in got.items():
        assert torch.equal(out, want[t]), (t, r)
    assert len(got) == 6


def test_cuda_graph_capture_of_a_grouped_call(pvb):
    """The fork and join are event record / wait pairs, which a capture follows onto the internal streams."""
    (m1, v1), (m2, v2) = _batches(2, 80)
    static_mask, static_vertex = m1.clone(), v1.clone()
    want1, want2 = _one_group(pvb, [(m1, v1)], 400)[0], _one_group(pvb, [(m2, v2)], 400)[0]
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        # the per-stream workspace and the internal streams are created outside the capture
        pvb.ransac_voting_layer_v3(static_mask, static_vertex, HN, inlier_thresh=0.99, seed=400)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            out = pvb.ransac_voting_layer_v3(static_mask, static_vertex, HN, inlier_thresh=0.99, seed=400)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want1)
    static_mask.copy_(m2)
    static_vertex.copy_(v2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want2)


def test_decode_v3_grouped(pvb):
    """pvb_decode_v3: the argmax front end reads the logits and writes the int64 mask per group."""
    mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=90, layout="planar")
    torch.manual_seed(3)
    seg = torch.stack([1.0 - mask.float(), mask.float()], dim=1)
    seg = (seg + 0.1 * torch.randn_like(seg)).contiguous()

    def run(groups):
        with _groups(groups):
            decode._decode_v3(seg, vertex, HN, 0.99, 5, 30000, 11, 0)
            ws = _ws()
            ws.zero_()
            m, out = decode._decode_v3(seg, vertex, HN, 0.99, 5, 30000, 11, 0)
            torch.cuda.synchronize()
            return m.clone(), out.clone(), ws.clone()

    a, b = run(0), run(1)
    assert torch.equal(a[0], b[0])
    _assert_same(a[1:], b[1:])
