"""Farthest-point sampling on the device (csrc/fps.cu) against the reference's indices: the fixture tests/golden/fps.npz,
the reference build oracle/_ref/libfps_ref.so where it exists, and the numpy restatement of its loop."""
import numpy as np
import pytest
import torch

import fps_cases

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def golden():
    return fps_cases.load_golden()


def _fps(pts, sn, init_center, start=None):
    x = torch.from_numpy(np.ascontiguousarray(pts, np.float32)[None]).to(DEV)
    from clean_pvnet_b200 import farthest_point_sampling_batch
    return farthest_point_sampling_batch(x, sn, init_center=init_center,
                                         starts=None if init_center else [start]).cpu().numpy()[0]


@pytest.mark.parametrize("kind", fps_cases.KINDS)
def test_equals_the_fixture(pvb, golden, kind):
    n = 0
    for k, pn, sn, seed, init_center, start, idxs in golden:
        if k != kind:
            continue
        got = _fps(fps_cases.cloud(k, pn, seed), sn, init_center, start)
        assert got.shape == (sn,)
        assert np.array_equal(got, idxs), (k, pn, sn, init_center, np.flatnonzero(got != idxs)[:5])
        n += 1
    assert n


def test_equals_the_reference_build(pvb):
    lib = fps_cases.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref/libfps_ref.so not built (no reference checkout)")
    for kind, pn, sn, seed in [("normal", pn, 64, 7 + pn) for pn in fps_cases.BOUNDARY_PN] + \
                              [("lattice", 24576, 500, 3), ("nanf", 40000, 64, 4), ("dup", 9000, 9003, 5)]:
        pts = fps_cases.cloud(kind, pn, seed)
        assert np.array_equal(_fps(pts, sn, True), fps_cases.ref_fps(lib, pts, sn, 1)), (kind, pn, sn)
        r = fps_cases.ref_fps(lib, pts, sn, 0)
        assert np.array_equal(_fps(pts, sn, False, int(r[0])), r), (kind, pn, sn)


def test_whole_cloud_at_capacity_boundaries(pvb):
    """sn = pn over clouds at the CTA and cluster boundaries: every point is selected, and the last ones tie at 0."""
    for pn in (511, 512, 513, 8191, 8192, 8193, 16385):
        pts = fps_cases.cloud("lattice", pn, 50 + pn)
        for init_center in (True, False):
            start = None if init_center else pn // 2
            got = _fps(pts, pn + 3, init_center, start)
            assert np.array_equal(got, fps_cases.fps_restated(pts, pn + 3, start)), (pn, init_center)


@pytest.mark.parametrize("init_center", [True, False])
def test_ragged_batch_equals_single_calls(pvb, init_center):
    rng = np.random.default_rng(11)
    counts = np.linspace(2000, 60000, 30).astype(np.int32)
    rng.shuffle(counts)
    n = int(counts.max())
    pts = np.full((len(counts), n, 3), np.nan, np.float32)        # rows past a cloud's count must not matter
    clouds = []
    for b, c in enumerate(counts):
        clouds.append(fps_cases.cloud("lattice" if b % 3 == 0 else "normal", int(c), 300 + b))
        pts[b, :c] = clouds[-1]
    starts = [int(rng.integers(c)) for c in counts]
    from clean_pvnet_b200 import farthest_point_sampling_batch
    got = farthest_point_sampling_batch(torch.from_numpy(pts).to(DEV), 8, init_center=init_center, counts=counts,
                                        starts=None if init_center else starts).cpu().numpy()
    assert got.shape == (len(counts), 8) and got.dtype == np.int32
    for b, c in enumerate(counts):
        one = _fps(clouds[b], 8, init_center, starts[b])
        assert np.array_equal(got[b], one), b
        assert np.array_equal(one, fps_cases.fps_restated(clouds[b], 8, None if init_center else starts[b])), b


def test_many_large_clouds_stream_through_the_workspace(pvb):
    """More clusters than fit at once: the launch narrows its clusters and streams the rest of each cloud."""
    counts = np.full(40, 70000, np.int32)
    counts[::5] = 65537
    pts = np.stack([fps_cases.cloud("normal", 70000, 900 + b) for b in range(len(counts))])
    from clean_pvnet_b200 import farthest_point_sampling_batch
    got = farthest_point_sampling_batch(torch.from_numpy(pts).to(DEV), 16, counts=counts).cpu().numpy()
    for b, c in enumerate(counts):
        assert np.array_equal(got[b], fps_cases.fps_restated(pts[b, :c], 16)), b


def test_fps_utils_surface(pvb):
    lib = fps_cases.ref_lib()
    pts = fps_cases.cloud("normal", 5000, 77).astype(np.float64)          # float64 in, rounded like the reference
    out = pvb.farthest_point_sampling(pts, 8, True)
    p32 = pts.astype(np.float32)
    assert out.dtype == np.float32 and out.shape == (8, 3)
    want = fps_cases.fps_restated(p32, 8) if lib is None else fps_cases.ref_fps(lib, p32, 8, 1)
    assert np.array_equal(out, p32[want])
    np.random.seed(5)
    out = pvb.farthest_point_sampling(pts, 8)
    np.random.seed(5)
    start = np.random.randint(5000)
    assert np.array_equal(out, p32[fps_cases.fps_restated(p32, 8, start)])
    assert pvb.farthest_point_sampling(pts, 0).shape == (0, 3)


def test_wrapper_rejects_bad_inputs(pvb):
    f = pvb.farthest_point_sampling_batch
    x = torch.zeros(2, 10, 3, device=DEV)
    with pytest.raises(RuntimeError, match=r"\[B,N,3\]"):
        f(torch.zeros(2, 10, 2, device=DEV), 4)
    with pytest.raises(RuntimeError, match=r"\[B,N,3\]"):
        f(torch.zeros(10, 3, device=DEV), 4)
    with pytest.raises(RuntimeError, match="sn"):
        f(x, -1)
    with pytest.raises(RuntimeError, match="one entry per cloud"):
        f(x, 4, counts=[10])
    with pytest.raises(RuntimeError, match="points"):
        f(x, 4, counts=[10, 11])
    with pytest.raises(RuntimeError, match="starts"):
        f(x, 4, init_center=False, starts=[0, 10])
    out = f(x.double(), 4)                                                  # other dtypes are converted
    assert out.dtype == torch.int32 and out.device == x.device and out.shape == (2, 4)
    assert f(x, 0).shape == (2, 0) and f(x[:0], 4).shape == (0, 4)


def test_side_stream_and_repeatability(pvb):
    pts = torch.from_numpy(fps_cases.cloud("lattice", 30000, 8)[None]).to(DEV).repeat(3, 1, 1)
    want = pvb.farthest_point_sampling_batch(pts, 64)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = pvb.farthest_point_sampling_batch(pts, 64)
    s.synchronize()
    assert torch.equal(got, want) and torch.equal(want[0], want[1]) and torch.equal(want[0], want[2])
