"""GPU: pass 1 of the pruned v3 vote classifies each tile's pixels once against the box of its 128 hypotheses (box_class,
csrc/vote.cu, DESIGN.md 4.2) and scores one hypothesis at a time only the undecided ones.

Bars: keypoints bit-identical to debug=True, and every hypothesis the passes scored has debug=True's count
(test_gpu_prune._compare, test_gpu_vote_list._check).  The forced cases read the kernel's own per-box counters
(pvb_set_pass1_stats) to check that pass 1 took the path each is meant to force, and that the counters add up to pass 1's
tests.  test_gpu_vote_list.py's ray-intersection and distinct-hypothesis cases drive pass 1's exact path as well."""
import numpy as np
import pytest
import torch

import test_gpu_prune as tgp
import test_gpu_vote_list as tvl

pytestmark = pytest.mark.gpu

HN, THRESH = 512, 0.99


def _box_stats(pvb, mask, vertex, seed):
    """pass 1's counters of the pruned call [resolved per box as inliers, resolved per box, scored one by one], checked
    against the call's pass-1 tests (list length x selected pixels); then pruned == full"""
    from clean_pvnet_b200 import _lib
    lib = _lib.load()
    stats = torch.zeros(3, dtype=torch.int64, device="cuda")
    _lib.check(lib.pvb_set_pass1_stats(stats.data_ptr()))
    try:
        _, views, lists, lens, _ = tgp._pruned(pvb, mask, vertex, HN, seed=seed)
    finally:
        _lib.check(lib.pvb_set_pass1_stats(None))
    s = stats.cpu().numpy()
    tn = np.maximum(views["tn"].cpu().numpy().astype(np.int64), 0)
    assert s[0] <= s[1]
    assert s[1] + s[2] == int((lens[0].astype(np.int64) * tn[:, None]).sum()), "the counters miss tests of pass 1"
    tvl._check(pvb, mask, vertex, seed)
    return s


def test_all_certain_clean_field(pvb):
    """Noise-free directions: every hypothesis sits on the keypoint, the box is ulps wide, and (nearly) every pixel is a
    certain inlier"""
    from clean_pvnet_b200 import synth
    mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=101, B=4, noise_deg=0.0, outlier_frac=0.0)
    s = _box_stats(pvb, mask, vertex, 102)
    assert s[0] > 0.95 * (s[1] + s[2]), s


def test_all_uncertain_random_field(pvb):
    """Random directions: pass 1's hypotheses spread over the image, so the box straddles the cone edges of most pixels
    and they are scored one hypothesis at a time; only pixels pointing away from the whole box are decided (outliers)"""
    from clean_pvnet_b200 import synth
    cfg = dict(synth.CONFIGS["cfg2"], random_field=True)
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=111, B=4)
    s = _box_stats(pvb, mask, vertex, 112)
    assert s[2] > 0.75 * (s[1] + s[2]), s


def test_bad_vectors_mix_both_paths(pvb):
    """Zero, NaN, infinite and huge vectors in a cfg-2 field: pixels that never vote are resolved as outliers, pixels
    outside the analysed domain are scored one by one (and decided exactly), the rest go either way"""
    from clean_pvnet_b200 import synth
    mask, vertex, _ = synth.make_inputs("cfg2", device="cuda", seed=81, B=4)
    vertex = vertex.clone()
    g = torch.Generator(device="cuda").manual_seed(82)
    fg = mask.nonzero()
    for i, val in enumerate([(0.0, 0.0), (float("nan"), 1.0), (float("inf"), 0.0), (1e30, -1e30)]):
        pick = fg[torch.randint(0, fg.shape[0], (3000,), generator=g, device="cuda")]
        vertex[pick[:, 0], pick[:, 1], pick[:, 2], i] = torch.tensor(val, device="cuda")
    s = _box_stats(pvb, mask, vertex, 83)
    assert s[0] > 0 and s[1] > s[0] and s[2] > 0, s


@pytest.mark.parametrize("thresh", [0.5, 0.9, 0.99, 0.999])
def test_cfg2_thresholds(pvb, thresh):
    mask, vertex, _ = tgp._inputs("cfg2", 1236)
    tgp._compare(pvb, mask, vertex, HN, thresh=thresh, seed=1236)


def test_cfg4_shaped_batch(pvb):
    mask, vertex, _ = tgp._inputs("cfg4", 1237, B=8)
    tgp._compare(pvb, mask, vertex, HN, seed=1237)


def test_uneven_grouped_split(pvb):
    """13 images run as groups of 6 and 7"""
    from clean_pvnet_b200 import synth
    cfg = dict(synth.CONFIGS["cfg2"], B=13)
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=1238)
    tgp._compare(pvb, mask, vertex, HN, seed=1238)
