"""GPU tests of the CenterNet heatmap loss (csrc/ct_loss.cu through clean_pvnet_b200.ct_loss):
  - the target equals the datasets' draw_umich_gaussian heatmap bit for bit (the stored fixture, the numpy restatement
    at B 1, 4 and 32 with 0 to 20 objects, and every (r, dx, dy) for r <= 64);
  - the gradient equals CUDA torch autograd of the trainer's expression on the dense target bit for bit, including an
    upstream gradient != 1, NaN / inf and clamp-saturated logits, a batch without objects and channels-last logits;
  - the loss is within one fp32 ulp of the same chain on float64 sums, and close to torch's fp32 sums;
  - reproducibility, no host synchronisation, a side-stream thread, DataParallel and one SGD step end to end."""
import os
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from ct_target_cases import case_images, restate_batch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ct_target.npz")
DEV = torch.device("cuda", 0)


def _bits_equal(a, b):
    """Equal bit for bit, except that any NaN equals any NaN (payloads are not part of the contract)."""
    a, b = a.detach(), b.detach()
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    return torch.equal(a[~na].contiguous().view(torch.int32), b[~nb].contiguous().view(torch.int32))


def _objects(B, M, C, H, W, seed, rmax=None, junk=False):
    """Random padded [B,M] objects: each image holds 0..M of them (ct_01 = 1), radii up to rmax, centres anywhere on
    the image.  junk: padding rows carry garbage values (only ct_01 marks them) and a few real rows have a class or
    centre out of range."""
    rng = np.random.default_rng(seed)
    rmax = rmax if rmax is not None else max(H, W) // 3
    ind = rng.integers(0, H * W, (B, M)).astype(np.int64)
    rad = rng.integers(0, rmax + 1, (B, M)).astype(np.int32)
    cls = rng.integers(0, C, (B, M)).astype(np.int64)
    n = rng.integers(0, M + 1, B) if M else np.zeros(B, np.int64)
    c01 = (np.arange(M)[None, :] < n[:, None]).astype(np.float32)
    if not junk:
        ind[c01 == 0], rad[c01 == 0], cls[c01 == 0] = 0, 0, 0
    else:
        if M >= 3:
            cls[:, 1] = C + 3
            ind[:, 2] = H * W + 5
            rad[0, 0] = -1
    return ind, rad, cls, c01


def _dev(*arrays):
    return [torch.from_numpy(a).to(DEV) for a in arrays]


# ---- target -----------------------------------------------------------------------------------------------------------

def test_target_equals_fixture(pvb):
    z = np.load(GOLDEN)
    for c, (B, C, H, W, _) in enumerate(case_images()):
        objs = _dev(z[f"ct_ind{c}"], z[f"ct_radius{c}"], z[f"ct_cls{c}"], z[f"ct_01{c}"])
        got = pvb.ct_target_batch(*objs, C, H, W)
        assert torch.equal(got, torch.from_numpy(z[f"ct_hm{c}"]).to(DEV)), c


@pytest.mark.parametrize("B", [1, 4, 32])
@pytest.mark.parametrize("M", [0, 1, 7, 20])
@pytest.mark.parametrize("HW", [(104, 128), (136, 184)])
def test_target_equals_restatement(pvb, B, M, HW):
    H, W = HW
    C = 30
    ind, rad, cls, c01 = _objects(B, M, C, H, W, seed=B * 100 + M + H, junk=True)
    got = pvb.ct_target_batch(*_dev(ind, rad, cls, c01), C, H, W)
    assert torch.equal(got, torch.from_numpy(restate_batch(ind, rad, cls, c01, C, H, W)).to(DEV))


def test_every_radius_offset_pair_up_to_64(pvb):
    """One image per radius r <= 64 with the object at the centre of a 129 x 129 image: every (dx, dy) in its window."""
    R = 64
    B, S = R + 1, 2 * R + 1
    ind = np.full((B, 1), R * S + R, np.int64)
    rad = np.arange(B, dtype=np.int32)[:, None]
    cls, c01 = np.zeros((B, 1), np.int64), np.ones((B, 1), np.float32)
    got = pvb.ct_target_batch(*_dev(ind, rad, cls, c01), 1, S, S)
    want = restate_batch(ind, rad, cls, c01, 1, S, S)
    assert torch.equal(got, torch.from_numpy(want).to(DEV))
    assert (want[:, 0, R, R] == 1).all() and (want > 0).sum() > 100000


# ---- the reference expression -----------------------------------------------------------------------------------------

def _reference_loss(logits, ct_hm):
    """lib/train/trainers/ct.py:20 (net_utils.FocalLoss on net_utils.sigmoid), verbatim on CUDA tensors."""
    pred = torch.clamp(logits.sigmoid(), min=1e-4, max=1 - 1e-4)
    gt = ct_hm
    pos_inds = gt.eq(1).float()
    neg_inds = gt.lt(1).float()
    neg_weights = torch.pow(1 - gt, 4)
    loss = 0
    pos_loss = torch.log(pred) * torch.pow(1 - pred, 2) * pos_inds
    neg_loss = torch.log(1 - pred) * torch.pow(pred, 2) * neg_weights * neg_inds
    num_pos = pos_inds.float().sum()
    pos_loss = pos_loss.sum()
    neg_loss = neg_loss.sum()
    if num_pos == 0:
        loss = loss - neg_loss
    else:
        loss = loss - (pos_loss + neg_loss) / num_pos
    return loss


def _logits(B, C, H, W, seed, layout="contiguous", scale=2.5):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.randn(B, C, H, W, generator=g) * scale).to(DEV)
    if layout == "channels_last":
        x = x.contiguous(memory_format=torch.channels_last)
    return x


CASES = {
    "plain":         dict(),
    "grad_out_3":    dict(scale=3.0),
    "odd_scale":     dict(scale=-0.7),
    "channels_last": dict(layout="channels_last"),
    "saturated":     dict(logit_scale=40.0),
    "nan_inf":       dict(poison=True),
    "no_objects":    dict(M=0),
    "all_padding":   dict(all_padding=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_gradient_is_autograd_bit_for_bit(pvb, case):
    cfg = CASES[case]
    B, C, H, W, M = 3, 30, 40, 52, cfg.get("M", 12)
    ind, rad, cls, c01 = _objects(B, M, C, H, W, seed=200 + list(CASES).index(case), rmax=9)
    if cfg.get("all_padding"):
        c01[:] = 0
    dense = torch.from_numpy(restate_batch(ind, rad, cls, c01, C, H, W)).to(DEV)
    objs = _dev(ind, rad, cls, c01)
    x = _logits(B, C, H, W, seed=7, layout=cfg.get("layout", "contiguous"), scale=cfg.get("logit_scale", 2.5))
    if cfg.get("poison"):
        with torch.no_grad():
            pos = (dense == 1).nonzero()[:2].tolist()
            x[pos[0][0], pos[0][1], pos[0][2], pos[0][3]] = float("nan")
            x[pos[1][0], pos[1][1], pos[1][2], pos[1][3]] = float("inf")
            x[0, 3, 5, 7], x[1, 4, 6, 8], x[2, 5, 7, 9] = float("-inf"), float("nan"), float("inf")
    scale = cfg.get("scale", 1.0)
    a = x.detach().clone().requires_grad_()
    ref = _reference_loss(a, dense)
    (ref * scale).backward()
    b = x.detach().clone().requires_grad_()
    got = pvb.ct_focal_loss(b, *objs)
    (got * scale).backward()
    assert _bits_equal(b.grad, a.grad)
    if cfg.get("poison"):
        assert torch.isnan(ref) and torch.isnan(got)
    else:
        r, g = float(ref.detach()), float(got.detach())
        assert abs(g - r) <= 1e-5 * abs(r), (g, r)
    if case in ("no_objects", "all_padding"):
        assert not (dense == 1).any()


def test_other_dtypes_are_refused(pvb):
    objs = _dev(*_objects(1, 3, 4, 8, 8, seed=0))
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        with pytest.raises(RuntimeError, match="float32"):
            pvb.ct_focal_loss(torch.zeros(1, 4, 8, 8, dtype=dt, device=DEV), *objs)
    with pytest.raises(RuntimeError, match=r"B = 2"):
        pvb.ct_focal_loss(torch.zeros(2, 4, 8, 8, device=DEV), *objs)


# ---- forward ----------------------------------------------------------------------------------------------------------

def _ulps(a, b):
    ia = np.array([a], np.float32).view(np.int32)[0]
    ib = np.array([b], np.float32).view(np.int32)[0]
    return abs(int(ia) - int(ib))


@pytest.mark.parametrize("B,H,W,seed", [(32, 104, 128, 1), (32, 136, 184, 2), (4, 104, 128, 3), (4, 136, 184, 4)])
def test_forward_against_float64_and_torch(pvb, B, H, W, seed):
    C, M = 30, 20
    ind, rad, cls, c01 = _objects(B, M, C, H, W, seed=seed, rmax=31)
    objs = _dev(ind, rad, cls, c01)
    t = pvb.ct_target_batch(*objs, C, H, W)               # == the restatement (test_target_equals_restatement)
    x = _logits(B, C, H, W, seed=seed)
    got = float(pvb.ct_focal_loss(x, *objs))
    pred = torch.clamp(x.sigmoid(), min=1e-4, max=1 - 1e-4)
    pos = (torch.log(pred) * torch.pow(1 - pred, 2) * t.eq(1).float()).double().sum()
    neg = (torch.log(1 - pred) * torch.pow(pred, 2) * torch.pow(1 - t, 4) * t.lt(1).float()).double().sum()
    n = int(t.eq(1).sum())
    pf, nf = np.float32(float(pos)), np.float32(float(neg))
    want = np.float32(0) - nf if n == 0 else np.float32(0) - np.float32((pf + nf) / np.float32(n))
    assert n > 0 and _ulps(got, want) <= 1, (got, want)
    ref = float(_reference_loss(x, t))
    rel = abs(got - ref) / abs(ref)
    print(f"[ct_loss] B={B} {H}x{W}: |fused - torch fp32| / torch = {rel:.3e} ({_ulps(got, ref)} ulp)")
    assert rel <= 1e-5


# ---- reproducibility, syncs, threads ----------------------------------------------------------------------------------

def _run_once(pvb, x, objs, scale=1.0):
    p = x.detach().clone().requires_grad_()
    loss = pvb.ct_focal_loss(p, *objs)
    (loss * scale).backward()
    return loss.detach(), p.grad


def test_bitwise_reproducible_and_sync_free(pvb):
    B, C, H, W, M = 32, 30, 104, 128, 20
    objs = _dev(*_objects(B, M, C, H, W, seed=21))
    x = _logits(B, C, H, W, seed=21)
    l1, g1 = _run_once(pvb, x, objs)
    p = x.clone().requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = pvb.ct_focal_loss(p, *objs)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _bits_equal(loss.detach(), l1) and _bits_equal(p.grad, g1)
    l2, g2 = _run_once(pvb, x, objs)
    assert _bits_equal(l2, l1) and _bits_equal(g2, g1)


def test_side_stream_in_a_thread(pvb):
    B, C, H, W, M = 4, 30, 104, 128, 12
    objs = _dev(*_objects(B, M, C, H, W, seed=31))
    x = _logits(B, C, H, W, seed=31)
    l1, g1 = _run_once(pvb, x, objs, scale=1.5)
    torch.cuda.synchronize()
    out = {}

    def work():
        s = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(s):
            out["r"] = _run_once(pvb, x, objs, scale=1.5)
        s.synchronize()

    t = threading.Thread(target=work)
    t.start()
    t.join()
    assert _bits_equal(out["r"][0], l1) and _bits_equal(out["r"][1], g1)


class _Head(torch.nn.Module):
    """A small conv head with the detector's outputs: 'ct_hm' (C channels) and 'wh' (2)."""

    def __init__(self, C, seed):
        super().__init__()
        torch.manual_seed(seed)
        self.conv = torch.nn.Conv2d(3, C + 2, 3, padding=1)
        self.C = C

    def forward(self, inp):
        out = self.conv(inp)
        return {'ct_hm': out[:, :self.C], 'wh': out[:, self.C:]}


def _batch(B, C, H, W, M, seed):
    ind, rad, cls, c01 = _objects(B, M, C, H, W, seed=seed, rmax=8)
    g = torch.Generator().manual_seed(seed)
    wh = torch.rand(B, M, 2, generator=g) * 20 * torch.from_numpy(c01)[..., None]
    batch = {'inp': torch.randn(B, 3, H, W, generator=g).to(DEV), 'wh': wh.to(DEV), 'meta': {}}
    batch.update(zip(('ct_ind', 'ct_radius', 'ct_cls', 'ct_01'), _dev(ind, rad, cls, c01)))
    dense = torch.from_numpy(restate_batch(ind, rad, cls, c01, C, H, W)).to(DEV)
    return batch, dense


def test_network_wrapper_inside_data_parallel(pvb):
    C = 30
    batch, _ = _batch(4, C, 48, 64, 10, seed=41)
    head = _Head(C, seed=1).to(DEV)
    w = pvb.CtNetworkWrapper(head)
    _, loss1, stats1, _ = w(batch)
    loss1.backward()
    g1 = head.conv.weight.grad.clone()
    head.zero_grad(set_to_none=True)
    dp = torch.nn.DataParallel(w, device_ids=[0])
    _, loss2, stats2, _ = dp(batch)
    loss2.mean().backward()
    assert set(stats2) == {'ct_loss', 'wh_loss', 'loss'}
    assert _bits_equal(loss2.reshape(()), loss1.reshape(()))
    assert _bits_equal(stats2['ct_loss'].reshape(()), stats1['ct_loss'].reshape(()))
    assert _bits_equal(head.conv.weight.grad, g1)


def test_one_sgd_step_equals_the_reference_trainer(pvb):
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    C = 30
    batch, dense = _batch(4, C, 48, 64, 10, seed=51)

    def step(head, loss_fn):
        opt = torch.optim.SGD(head.parameters(), lr=0.1, momentum=0.9)
        opt.zero_grad()
        loss_fn(head).backward()
        opt.step()
        return [p.detach().clone() for p in head.parameters()]

    def reference(head):                     # lib/train/trainers/ct.py, forward, on the dense heatmap
        output = head(batch['inp'])
        loss = 0
        loss += _reference_loss(output['ct_hm'], dense)
        feat = output['wh'].permute(0, 2, 3, 1).contiguous()
        feat = feat.view(feat.size(0), -1, feat.size(3))
        ind = batch['ct_ind'].unsqueeze(2).expand(batch['ct_ind'].size(0), batch['ct_ind'].size(1), feat.size(2))
        feat = feat.gather(1, ind)
        weight = batch['ct_01'].unsqueeze(2)
        wh_loss = F.smooth_l1_loss(feat * weight, batch['wh'] * weight, reduction='sum')
        wh_loss = wh_loss / (weight.sum() * feat.size(2) + 1e-4)
        loss += 0.1 * wh_loss
        return loss

    want = step(_Head(C, seed=2).to(DEV), reference)
    got = step(_Head(C, seed=2).to(DEV), lambda head: pvb.CtNetworkWrapper(head)(batch)[1])
    for a, b in zip(got, want):
        assert _bits_equal(a, b)
