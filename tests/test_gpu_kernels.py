"""GPU parity, kernel boundary: the C-ABI twins of the reference extension and the layer's vote
kernel against the CPU oracle.  Hypotheses must be bit-equal, inlier bytes / counts equal."""
import numpy as np
import pytest
import torch

from util import bits_equal, cuda, field_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tn,vn,hn,seed", [(2000, 3, 128, 0), (517, 1, 33, 1), (4096, 9, 512, 2), (64, 17, 8, 3)])
def test_generate_hypothesis_bit_exact(pvb, oracle, tn, vn, hn, seed):
    direct, coords, idxs, _ = field_case(tn, vn, hn, seed)
    want = oracle.generate_hypothesis(direct, coords, idxs)
    d, c, i = cuda(direct, coords, idxs)
    got = pvb.ransac_voting.generate_hypothesis(d, c, i).cpu().numpy()
    assert got.shape == want.shape
    assert bits_equal(got, want)
    assert tuple(got[0, 0]) == (0.0, 0.0)          # t0 == t1


def test_generate_hypothesis_near_parallel(pvb, oracle):
    # determinants straddling the 1e-6 double-precision cut (.cu:42-43)
    rng = np.random.default_rng(5)
    n = 2000
    coords = rng.integers(0, 640, size=(2 * n, 2)).astype(np.float32)
    a0 = rng.uniform(0, 2 * np.pi, size=n)
    delta = rng.choice([0.0, 5e-7, 8e-7, 9.5e-7, 1.05e-6, 1.2e-6, 2e-6, 1e-5, 1e-3], size=n) * rng.choice([-1, 1], size=n)
    a1 = a0 + delta + rng.choice([0.0, np.pi], size=n)
    ang = np.stack([a0, a1], axis=1).reshape(-1)
    direct = np.stack([np.cos(ang), np.sin(ang)], axis=-1).astype(np.float32)[:, None, :]
    idxs = np.stack([np.arange(0, 2 * n, 2), np.arange(1, 2 * n, 2)], axis=1).astype(np.int32)[:, None, :]
    want = oracle.generate_hypothesis(direct, coords, idxs)
    got = pvb.ransac_voting.generate_hypothesis(*cuda(direct, coords, idxs)).cpu().numpy()
    assert bits_equal(got, want)
    zero = (want == 0).all(axis=-1).mean()
    assert 0.05 < zero < 0.95                      # both branches exercised


@pytest.mark.parametrize("thresh", [0.99, 0.999])
def test_voting_for_hypothesis_bytes(pvb, oracle, thresh):
    direct, coords, idxs, _ = field_case(1500, 3, 64, 4)
    hyp = oracle.generate_hypothesis(direct, coords, idxs)
    want = np.zeros((64, 3, 1500), dtype=np.uint8)
    oracle.voting_for_hypothesis(direct, coords, hyp, want, thresh)
    d, c, h = cuda(direct, coords, hyp)
    got = torch.full((64, 3, 1500), 0, dtype=torch.uint8, device="cuda")
    got[5] = 9                                     # bytes that are not inliers must stay untouched
    pvb.ransac_voting.voting_for_hypothesis(d, c, h, got, thresh)
    got = got.cpu().numpy()
    assert np.array_equal(got[np.arange(64) != 5], want[np.arange(64) != 5])
    assert np.array_equal(got[5] == 1, want[5] == 1) and set(np.unique(got[5])) <= {1, 9}
    assert want.sum() > 1000


@pytest.mark.parametrize("tn,vn,hn,seed,thresh", [
    (3000, 3, 128, 0, 0.99), (3000, 3, 256, 1, 0.999), (1111, 2, 700, 2, 0.99), (5000, 9, 512, 3, 0.99),
    (300, 1, 2048, 4, 0.9), (2500, 4, 64, 5, 0.5), (800, 2, 100, 6, 0.05)])
def test_vote_count_matches_oracle(pvb, oracle, tn, vn, hn, seed, thresh):
    direct, coords, idxs, _ = field_case(tn, vn, hn, seed)
    hyp = oracle.generate_hypothesis(direct, coords, idxs)
    want = oracle.vote_count(direct, coords, hyp, thresh)
    got = pvb.ransac_voting.vote_count(*cuda(direct, coords, hyp), thresh).cpu().numpy()
    assert np.array_equal(got, want)
    assert want.max() > 10


@pytest.mark.parametrize("thresh", [0.0, -0.5, 1.0, 1.5, float(np.nextafter(np.float32(1), np.float32(0)))])
def test_vote_count_threshold_outside_cone_domain(pvb, oracle, thresh):
    # thresholds <= 0 or >= 1 have no cone formulation: every test takes the exact path
    direct, coords, idxs, _ = field_case(700, 2, 96, 8)
    hyp = oracle.generate_hypothesis(direct, coords, idxs)
    want = oracle.vote_count(direct, coords, hyp, thresh)
    got = pvb.ransac_voting.vote_count(*cuda(direct, coords, hyp), thresh).cpu().numpy()
    assert np.array_equal(got, want)


def test_vote_count_adversarial(pvb, oracle):
    """Borderline geometry: hypotheses on pixels, on the cone boundary, far away, non-finite;
    zero / tiny / huge / non-finite direction vectors; non-integer coordinates."""
    rng = np.random.default_rng(11)
    tn, vn, hn = 2048, 2, 512
    thresh = 0.99
    coords = rng.uniform(0, 640, size=(tn, 2)).astype(np.float32)
    coords[: tn // 2] = np.round(coords[: tn // 2])
    ang = rng.uniform(0, 2 * np.pi, size=(tn, vn))
    direct = np.stack([np.cos(ang), np.sin(ang)], axis=-1).astype(np.float32)
    scale = rng.choice([1.0, 1e-7, 1e-6, 1.1e-6, 1e-3, 1e4, 1e19, 0.0], size=(tn, vn, 1), p=[.6, .05, .05, .05, .05, .1, .05, .05])
    direct = (direct * scale).astype(np.float32)
    direct[3, 0] = [np.nan, 1.0]
    direct[4, 1] = [np.inf, 0.0]
    hyp = rng.uniform(-200, 900, size=(hn, vn, 2)).astype(np.float32)
    # exactly on pixels, and a hair off
    hyp[:64, 0] = coords[:64]
    hyp[64:128, 0] = coords[64:128] + np.float32(5e-7)
    # on the cone boundary of some pixel: pixel + r * (direction rotated by +-acos(thresh))
    th = np.arccos(np.float32(thresh))
    for j in range(128, 384):
        t = rng.integers(0, tn)
        k = j % vn
        a = np.arctan2(direct[t, k, 1], direct[t, k, 0]) + rng.choice([-1, 1]) * th * rng.choice([1.0, 1 + 1e-7, 1 - 1e-7, 1 + 1e-5])
        r = rng.choice([0.5, 3.0, 50.0, 700.0, 1e5])
        hyp[j, k] = coords[t] + r * np.array([np.cos(a), np.sin(a)], dtype=np.float64)
    hyp[384:400] *= 1e6
    hyp[400:404] *= 1e20
    hyp[404, 0] = [np.nan, 3.0]
    hyp[405, 1] = [np.inf, -np.inf]
    hyp[406] = 0.0
    with np.errstate(all="ignore"):
        want = oracle.vote_count(direct, coords, hyp, thresh)
    got = pvb.ransac_voting.vote_count(*cuda(direct, coords, hyp), thresh).cpu().numpy()
    assert np.array_equal(got, want)


@pytest.fixture
def vote_variant():
    """Force one vote kernel (include/pvnet_vote_b200.h, pvb_set_tuning) for the duration of a test."""
    from clean_pvnet_b200 import _lib
    lib = _lib.load()

    def force(v):
        _lib.check(lib.pvb_set_tuning(0, v))
    yield force
    _lib.check(lib.pvb_set_tuning(0, 0))


@pytest.mark.parametrize("variant", [1, 2, 3])
@pytest.mark.parametrize("tn,vn,hn,seed,thresh", [
    (1500, 2, 24, 20, 0.99), (2100, 3, 64, 21, 0.99), (3000, 2, 130, 22, 0.999), (1111, 2, 512, 23, 0.99),
    (2500, 1, 520, 24, 0.9), (1030, 2, 1100, 25, 0.99), (17, 1, 8, 26, 0.99), (1024, 1, 64, 27, 0.5)])
def test_every_vote_kernel_matches_oracle(pvb, oracle, vote_variant, variant, tn, vn, hn, seed, thresh):
    """Every launch shape of the vote kernel (above 256 hypotheses, pixel tile 1024 / 256 / 512 for variants 1 / 2 / 3,
    otherwise 512; 1, 2 or 4 hypotheses per thread; 1, 2 or 4 warp teams per CTA) at hypothesis counts on both sides of
    each switch-over, with partial slices and partial pixel tiles."""
    direct, coords, idxs, _ = field_case(tn, vn, hn, seed)
    hyp = oracle.generate_hypothesis(direct, coords, idxs)
    want = oracle.vote_count(direct, coords, hyp, thresh)
    vote_variant(variant)
    got = pvb.ransac_voting.vote_count(*cuda(direct, coords, hyp), thresh).cpu().numpy()
    assert np.array_equal(got, want)


@pytest.mark.parametrize("variant", [1, 2, 3])
def test_every_vote_kernel_adversarial(pvb, oracle, vote_variant, variant):
    """The adversarial case above under each kernel, plus hypotheses/pixels that force the exact path wholesale."""
    rng = np.random.default_rng(12)
    tn, vn, hn = 1500, 2, 200
    coords = np.round(rng.uniform(0, 640, size=(tn, 2))).astype(np.float32)
    ang = rng.uniform(0, 2 * np.pi, size=(tn, vn))
    direct = np.stack([np.cos(ang), np.sin(ang)], axis=-1).astype(np.float32)
    scale = rng.choice([1.0, 1e-7, 1.1e-6, 1e4, 1e19, 0.0], size=(tn, vn, 1), p=[.7, .05, .05, .1, .05, .05])
    direct = (direct * scale).astype(np.float32)
    direct[5, 0] = [np.nan, 1.0]
    direct[6, 1] = [np.inf, 0.0]
    coords[7] = [1e7, -3e6]          # far outside its tile's box: that tile's records go the exact way
    hyp = rng.uniform(-200, 900, size=(hn, vn, 2)).astype(np.float32)
    hyp[:32, 0] = coords[:32]
    th = np.arccos(np.float32(0.99))
    for j in range(32, 160):
        t = rng.integers(0, tn)
        k = j % vn
        a = np.arctan2(direct[t, k, 1], direct[t, k, 0]) + rng.choice([-1, 1]) * th * rng.choice([1.0, 1 + 1e-7, 1 - 1e-7])
        r = rng.choice([0.5, 3.0, 50.0, 700.0, 1e5])
        hyp[j, k] = coords[t] + r * np.array([np.cos(a), np.sin(a)], dtype=np.float64)
    hyp[160:170] *= 1e6
    hyp[170:174] *= 1e20
    hyp[174, 0] = [np.nan, 3.0]
    hyp[175, 1] = [np.inf, -np.inf]
    with np.errstate(all="ignore"):
        want = oracle.vote_count(direct, coords, hyp, 0.99)
    vote_variant(variant)
    got = pvb.ransac_voting.vote_count(*cuda(direct, coords, hyp), 0.99).cpu().numpy()
    assert np.array_equal(got, want)


def _ulp_ring(x, y):
    """(x, y), and its float32 neighbours one ulp away in x, in y and in both."""
    up, dn = np.float32(np.inf), np.float32(-np.inf)
    xs = [np.float32(x), np.nextafter(np.float32(x), up), np.nextafter(np.float32(x), dn)]
    ys = [np.float32(y), np.nextafter(np.float32(y), up), np.nextafter(np.float32(y), dn)]
    return np.array([(a, b) for a in xs for b in ys], dtype=np.float32)


@pytest.mark.parametrize("variant,hn,tile", [(1, 300, 1024), (2, 300, 256), (3, 300, 512), (1, 64, 512)])
def test_vote_count_single_point_tiles(pvb, oracle, vote_variant, variant, hn, tile):
    """tn = 2*tile + 1: the last tile holds one pixel, at small integer coordinates, and tile 1 has all its pixels at one
    position.  Such tiles have a bounding box of ~0, so the guard band alone is tiny; hypotheses 1 ulp from those
    positions (0 < |h-c| < 1e-6: the reference's norm cut) and exactly on them must still count as the reference does."""
    rng = np.random.default_rng(variant * 1000 + hn)
    tn, vn = 2 * tile + 1, 4
    direct, coords, idxs, _ = field_case(tn, vn, hn, seed=variant)
    hyp = oracle.generate_hypothesis(direct, coords, idxs)
    coords[-1] = (3, 5)
    coords[tile:2 * tile] = (7, 2)
    u = np.array([(1, 0), (0, 1), (-0.6, 0.8), (0.70710677, -0.70710677)], dtype=np.float32)
    direct[-1] = u                                   # per keypoint: which ulp neighbours lie inside the cone differs
    ang = rng.uniform(0, 2 * np.pi, tile)
    direct[tile:2 * tile] = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)[:, None, :]
    direct[tile:tile + 4] = u[None]                  # some of the shared-position pixels point at the ring exactly
    near = np.concatenate([_ulp_ring(3, 5), _ulp_ring(7, 2), _ulp_ring(0, 0), _ulp_ring(1, 15)])
    hyp[:len(near)] = near[:, None, :]
    want = oracle.vote_count(direct, coords, hyp, 0.99)
    vote_variant(variant)
    got = pvb.ransac_voting.vote_count(*cuda(direct, coords, hyp), 0.99).cpu().numpy()
    assert np.array_equal(got, want)
    assert (want[:len(near)] > 0).any() and want.max() > 10


def test_vote_count_empty_and_ragged(pvb, oracle):
    direct, coords, idxs, _ = field_case(257, 5, 129, 9)
    hyp = oracle.generate_hypothesis(direct, coords, idxs)
    assert np.array_equal(pvb.ransac_voting.vote_count(*cuda(direct, coords, hyp), 0.99).cpu().numpy(),
                          oracle.vote_count(direct, coords, hyp, 0.99))
    d, c, h = cuda(direct[:0], coords[:0], hyp)
    assert (pvb.ransac_voting.vote_count(d, c, h, 0.99) == 0).all()
    d, c, h = cuda(direct, coords, hyp[:0])
    assert pvb.ransac_voting.vote_count(d, c, h, 0.99).shape == (0, 5)


def test_vanishing_point_twins_bit_exact(pvb, oracle):
    direct, coords, idxs, _ = field_case(1500, 3, 96, 12)
    want = oracle.generate_hypothesis(direct, coords, idxs, vanishing_point=True)
    d, c, i = cuda(direct, coords, idxs)
    got = pvb.ransac_voting.generate_hypothesis_vanishing_point(d, c, i)
    assert bits_equal(got.cpu().numpy(), want)
    wi = np.zeros((96, 3, 1500), dtype=np.uint8)
    oracle.voting_for_hypothesis(direct, coords, want, wi, 0.999, vanishing_point=True)
    gi = torch.zeros((96, 3, 1500), dtype=torch.uint8, device="cuda")
    pvb.ransac_voting.voting_for_hypothesis_vanishing_point(d, c, got, gi, 0.999)
    assert np.array_equal(gi.cpu().numpy(), wi)
    assert wi.sum() > 1000


def test_input_checks_match_reference(pvb):
    d = torch.zeros(8, 2, 2, device="cuda")
    c = torch.zeros(8, 2, device="cuda")
    i = torch.zeros(4, 2, 2, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="contiguous"):
        pvb.ransac_voting.generate_hypothesis(d.transpose(0, 1).contiguous().transpose(0, 1), c, i)
    with pytest.raises(RuntimeError, match="CUDA"):
        pvb.ransac_voting.generate_hypothesis(d.cpu(), c, i)
    with pytest.raises(RuntimeError):
        pvb.ransac_voting.generate_hypothesis(d, c, i.long())
