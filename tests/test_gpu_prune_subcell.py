"""GPU: the pruned v3 vote's sub-cell records and its pass-2 refinement (csrc/prune.cu) against the numpy twin.

Wherever pruning runs: the sub-cell records equal prune_subcell_twin.subcell_records bit for bit (an empty one is its last word
alone); B(h) and B2(h) are >= the exact count of debug=True; pass 2 is exactly {h not in pass 1 : B(h) >= L and
B2(h) >= L} of the kernels' own bounds, L the best pass-1 count.  The bounds divide approximately (pseudo_angle), so
they equal the twin's, which divides with IEEE rounding, for all but a few hypotheses whose window end falls within
rounding of a bin edge: at least 99 % must agree, and the pass lists the twin's bounds give must then agree as well
except where a bound differs.  test_gpu_prune._compare checks the rest: keypoints, winners and every scored count
bit-identical to debug=True, and the cell records equal to the twin's."""
import numpy as np
import pytest
import torch

import test_gpu_prune as tgp
from prune_subcell_twin import pass_lists, subcell_records
from prune_twin import REC, F, cell_records, count_bound, prune_applies, prune_rotation

pytestmark = pytest.mark.gpu


def _regions(mask, vertex, hn, thresh):
    """prune_key, both lists and lengths, the sub-cell records and the sub-cell bounds of the last call on this
    workspace"""
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    lib = _lib.load()
    m, v = rv._check_inputs(mask, vertex)
    d = rv._make_desc(m, v, hn, thresh, 5, 30000, _lib.PVB_SELECT_BYTE, 0, 0, None)
    ws = rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)]
    L = _lib.PvbLayout()
    _lib.check(lib.pvb_workspace_layout(d, L))
    B, K = d.B, d.K
    sub_off = (L.prune_len + 2 * B * K * 4 + 255) // 256 * 256     # the sub-cell records follow prune_len
    nsub = B * K * L.prune_ncells * 4 * REC
    b2_off = (sub_off + 4 * nsub + 255) // 256 * 256                # then the sub-cell bounds
    assert b2_off + 4 * B * K * hn <= L.total

    def ints(off, n):
        return ws[off:off + 4 * n].view(torch.int32).cpu().numpy()
    key = ints(L.prune_key, B * K * hn).reshape(B, K, hn)
    lists = ints(L.prune_list, 2 * B * K * hn).reshape(2, B, K, hn)
    lens = ints(L.prune_len, 2 * B * K).reshape(2, B, K)
    sub = ints(sub_off, nsub).reshape(B, K, L.prune_ncells, 4, REC)
    b2 = ints(b2_off, B * K * hn).reshape(B, K, hn)
    return key, lists, lens, sub, b2


def _check(pvb, mask, vertex, hn, thresh=0.99, seed=1000):
    tgp._compare(pvb, mask, vertex, hn, thresh, seed=seed)
    B, H, W, K = vertex.shape[:4]
    assert prune_applies(thresh, hn, B, K)
    pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=thresh, seed=seed)
    torch.cuda.synchronize()
    key, lists, lens, sub, b2k = _regions(mask, vertex, hn, thresh)
    _, dbg = pvb.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=thresh, seed=seed, debug=True)
    from clean_pvnet_b200 import _lib, ransac_voting_gpu as rv
    views = rv._views(rv._workspaces[(mask.device.index, torch.cuda.current_stream().cuda_stream)],
                      rv._make_desc(*rv._check_inputs(mask, vertex), hn, thresh, 5, 30000, _lib.PVB_SELECT_BYTE,
                                    seed, 0, None), _lib.load())
    tn = views["tn"].cpu().numpy()
    xy, dirs = views["xy"].cpu().numpy(), views["dirs"].cpu().numpy()
    hyp, cnt = dbg["hyp"].cpu().numpy().astype(F), dbg["counts"].cpu().numpy()
    rot = prune_rotation(thresh)
    p2_len, agree, total = [], 0, 0
    for b in range(B):
        for k in range(K):
            n, c = tn[b], cnt[b, k]
            want_sub = subcell_records(xy[b, :n], dirs[b, k, :n], H, W)
            full = (want_sub[:, :, -1] >> 16) > 0
            bad = np.nonzero(((sub[b, k] != want_sub).any(-1) & full) | (sub[b, k, :, :, -1] != want_sub[:, :, -1]))
            assert bad[0].size == 0, f"image {b} keypoint {k}: sub-cells {list(zip(*bad))[:4]} differ from the twin"
            p1 = lists[0, b, k, :lens[0, b, k]]
            p2 = lists[1, b, k, :lens[1, b, k]]
            ok = np.abs(hyp[b, k]).sum(1) <= F(1e15)
            # the kernels' own bounds: safe, and pass 2 is what they select
            L = c[p1].max() if len(p1) else 0
            assert (key[b, k][p1] == -1).all() and np.count_nonzero(key[b, k] == -1) == len(p1)
            rest = key[b, k] >= 0
            assert (key[b, k][rest] >= c[rest]).all(), (b, k)
            cand = rest & (key[b, k] >= L) & ok
            if L > 0:
                assert (b2k[b, k][cand] >= c[cand]).all(), (b, k)
            keep = rest & (key[b, k] >= L) & (~ok | (b2k[b, k] >= L) | (L == 0))
            assert np.array_equal(p2, np.nonzero(keep)[0]), (b, k)
            # against the twin
            bnd = count_bound(hyp[b, k], cell_records(xy[b, :n], dirs[b, k, :n], H, W), n, rot)
            b2 = count_bound(hyp[b, k], want_sub.reshape(-1, REC), n, rot)
            same = (bnd == np.where(rest, key[b, k], bnd)) & (~cand | (L == 0) | (b2 == b2k[b, k]))
            agree += np.count_nonzero(same)
            total += len(same)
            t1, t2, _ = pass_lists(bnd, b2, c)
            if same.all():
                assert np.array_equal(p1, t1) and np.array_equal(p2, t2), (b, k)
            p2_len.append(len(p2))
    assert agree >= 0.99 * total, (agree, total)
    return np.array(p2_len)


@pytest.mark.parametrize("cfg,B", [("cfg2", 4), ("cfg3", 4), ("cfg4", 2), ("cfg5", 4)])
def test_subcells_production_shapes(pvb, cfg, B):
    from clean_pvnet_b200 import synth
    mask, vertex, _ = tgp._inputs(cfg, 1236, B=B)
    p2 = _check(pvb, mask, vertex, synth.CONFIGS[cfg]["hn"])
    if cfg == "cfg2":
        print(f"cfg2 pass-2 entries per (image, keypoint): mean {p2.mean():.1f} min {p2.min()} max {p2.max()}")


@pytest.mark.parametrize("thresh", [0.5, 0.9, 0.999])
def test_subcells_thresholds(pvb, thresh):
    mask, vertex, _ = tgp._inputs("cfg2", 21, B=4)
    _check(pvb, mask, vertex, 512, thresh=thresh, seed=22)


@pytest.mark.parametrize("H,W,hn", [(97, 141, 300), (111, 50, 129), (63, 65, 2048), (200, 129, 1024)])
def test_subcells_on_sub_cell_borders(pvb, H, W, hn):
    """image sides 1..15 mod 16: the last row and column of sub-cells lie partly outside the image"""
    from clean_pvnet_b200 import synth
    cfg = dict(B=8, H=H, W=W, K=4, hn=hn, fill=(0.3, 0.6), kind="blob")
    mask, vertex, _ = synth.make_inputs(cfg, device="cuda", seed=H + W)
    _check(pvb, mask, vertex, hn, seed=7)


def test_subcells_skipped_images_and_zero_vectors(pvb):
    """a skipped image and an image whose vectors are all zero (L = 0: pass 2 is every hypothesis not in pass 1)"""
    mask, vertex, _ = tgp._inputs("cfg2", 51, B=4)
    mask = mask.clone()
    mask[1] = 0
    vertex = vertex.clone()
    vertex[2] = 0.0
    p2 = _check(pvb, mask, vertex, 512, seed=52)
    assert (p2.reshape(4, -1)[2] == 512 - 128).all()
