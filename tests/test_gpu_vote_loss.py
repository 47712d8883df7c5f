"""GPU tests of the vote loss (csrc/loss.cu through clean_pvnet_b200.vote_loss):
  - the target field equals clean-pvnet's compute_vertex bit for bit (the stored fixture, then the numpy restatement at
    the sampler's extreme sizes, an odd size, B in {1, 3, 32} and K in {1, 9, 17});
  - the gradient equals CUDA torch autograd of the trainer's expression on the dense restated target bit for bit,
    including NaN / inf predictions, an empty mask, mask values 2 and 255 and strided predictions;
  - the loss is within one fp32 ulp of the same chain on a float64 sum of the terms, and close to torch's fp32 sum;
  - reproducibility, no host synchronisation, DataParallel and side-stream threads, and one SGD step end to end."""
import os
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from vote_target_cases import restate_vertex

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vote_target.npz")
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


def _inputs(B, H, W, K, seed, fill=0.3, values=(1,)):
    """(mask uint8 [B,H,W], kpt float64 [B,K,2]) on the host: about `fill` of the pixels foreground (value drawn from
    `values`), keypoints around and beyond the image."""
    rng = np.random.default_rng(seed)
    fg = rng.random((B, H, W)) < fill
    mask = np.where(fg, rng.choice(np.array(values, np.uint8), size=(B, H, W)), 0).astype(np.uint8)
    kpt = np.stack([rng.uniform(-0.2 * W, 1.2 * W, (B, K)), rng.uniform(-0.2 * H, 1.2 * H, (B, K))], -1)
    return mask, kpt


def _restate(mask, kpt):
    return np.stack([restate_vertex(m, k) for m, k in zip(mask, kpt)])


def _reference_loss(pred, mask, vertex):
    """lib/train/trainers/pvnet.py:25-27, verbatim on CUDA tensors."""
    weight = mask[:, None].float()
    vote_loss = F.smooth_l1_loss(pred * weight, vertex * weight, reduction='sum')
    return vote_loss / weight.sum() / vertex.size(1)


# ---- target -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64])
def test_target_equals_fixture(pvb, dtype):
    z = np.load(GOLDEN)
    for c in range(3):
        mask = torch.from_numpy(z[f"mask{c}"]).to(DEV)
        if dtype == torch.int8:
            mask = mask.to(torch.int16).to(dtype)        # 255 -> -1: still not 1, still no vector
        else:
            mask = mask.to(dtype)
        kpt = torch.from_numpy(z[f"kpt{c}"]).to(DEV)
        got = pvb.vote_target_batch(mask, kpt)
        assert _bits_equal(got, torch.from_numpy(z[f"vertex{c}"]).to(DEV)), c
        # a strided view of the same mask
        big = torch.zeros(mask.shape[0], mask.shape[1] + 3, mask.shape[2] + 5, dtype=dtype, device=DEV)
        big[:, 2:2 + mask.shape[1], 1:1 + mask.shape[2]] = mask
        view = big[:, 2:2 + mask.shape[1], 1:1 + mask.shape[2]]
        assert _bits_equal(pvb.vote_target_batch(view, kpt), got)


def test_target_bool_mask_and_float32_keypoints(pvb):
    mask, kpt = _inputs(2, 33, 47, 9, seed=5, values=(1, 2))
    k32 = kpt.astype(np.float32)
    want = _restate(mask != 0, k32)
    got = pvb.vote_target_batch(torch.from_numpy(mask != 0).to(DEV), torch.from_numpy(k32))
    assert _bits_equal(got, torch.from_numpy(want).to(DEV))


@pytest.mark.parametrize("B,H,W,K", [(1, 256, 256, 9), (1, 480, 640, 17), (3, 479, 641, 1), (3, 479, 641, 17),
                                     (32, 256, 256, 9), (32, 480, 640, 9)])
def test_target_equals_restatement(pvb, B, H, W, K):
    mask, kpt = _inputs(B, H, W, K, seed=B * 1000 + K, values=(1, 1, 1, 2, 255))
    got = pvb.vote_target_batch(torch.from_numpy(mask).to(DEV), torch.from_numpy(kpt).to(DEV))
    assert _bits_equal(got, torch.from_numpy(_restate(mask, kpt)).to(DEV))


# ---- gradient ---------------------------------------------------------------------------------------------------------

def _pred(B, K, H, W, seed, layout):
    """A leaf tensor and the fp32 [B,2K,H,W] prediction view of it the loss reads."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    if layout == "contiguous":
        leaf = (torch.randn(B, 2 * K, H, W, generator=g) * 1.5).to(DEV)
        return leaf.requires_grad_(), lambda t: t
    if layout == "channels_last":
        leaf = (torch.randn(B, 2 * K, H, W, generator=g) * 1.5).to(DEV).contiguous(memory_format=torch.channels_last)
        return leaf.requires_grad_(), lambda t: t
    leaf = (torch.randn(B, 2 * K + 5, H, W, generator=g) * 1.5).to(DEV)      # a channel slice, as output[:, :2K]
    return leaf.requires_grad_(), lambda t: t[:, 3:3 + 2 * K]


def _grads(pvb, leaf_data, view, mask, kpt, vertex, scale):
    a = leaf_data.detach().clone().requires_grad_()
    ref = _reference_loss(view(a), mask, vertex)
    (ref * scale).backward()
    b = leaf_data.detach().clone().requires_grad_()
    got = pvb.vote_loss(view(b), mask, kpt)
    (got * scale).backward()
    return ref, got, a.grad, b.grad


CASES = {
    "plain":         dict(values=(1,), layout="contiguous", scale=1.0),
    "grad_out_3":    dict(values=(1,), layout="contiguous", scale=3.0),
    "odd_scale":     dict(values=(1,), layout="contiguous", scale=-0.7),
    "values_2_255":  dict(values=(1, 1, 2, 255), layout="contiguous", scale=1.0),
    "channels_last": dict(values=(1,), layout="channels_last", scale=1.0),
    "channel_slice": dict(values=(1, 2), layout="slice", scale=2.0),
    "nan_inf":       dict(values=(1,), layout="contiguous", scale=1.0, poison=True),
    "empty_mask":    dict(values=(1,), layout="contiguous", scale=1.0, fill=0.0),
}


@pytest.mark.parametrize("mask_dtype", [torch.uint8, torch.int64, torch.bool])
@pytest.mark.parametrize("case", list(CASES))
def test_gradient_is_autograd_bit_for_bit(pvb, case, mask_dtype):
    cfg = CASES[case]
    B, H, W, K = 2, 61, 83, 9
    mask_np, kpt_np = _inputs(B, H, W, K, seed=100 + list(CASES).index(case), fill=cfg.get("fill", 0.3),
                              values=cfg["values"])
    if mask_dtype == torch.bool:
        mask_np = mask_np != 0
    mask = torch.from_numpy(mask_np).to(DEV).to(mask_dtype)
    kpt = torch.from_numpy(kpt_np).to(DEV)
    vertex = torch.from_numpy(_restate(mask_np, kpt_np)).to(DEV)
    leaf, view = _pred(B, K, H, W, seed=11, layout=cfg["layout"])
    if cfg.get("poison"):
        with torch.no_grad():
            p = view(leaf)
            m = mask_np.astype(bool)
            inside, outside = np.argwhere(m)[:2], np.argwhere(~m)[:2]
            p[inside[0][0], 0, inside[0][1], inside[0][2]] = float("nan")
            p[inside[1][0], 3, inside[1][1], inside[1][2]] = float("inf")
            p[outside[0][0], 5, outside[0][1], outside[0][2]] = float("-inf")
            p[outside[1][0], 7, outside[1][1], outside[1][2]] = float("nan")
    ref, got, gref, ggot = _grads(pvb, leaf, view, mask, kpt, vertex, cfg["scale"])
    assert _bits_equal(ggot, gref)
    if case in ("nan_inf", "empty_mask"):
        assert torch.isnan(ref) and torch.isnan(got)                  # the reference's NaN loss, kept
        if case == "empty_mask":
            assert torch.isnan(ggot).all()                           # (g / 2K) / 0 = inf, then 0 * inf
    else:
        assert abs(float(got.detach()) - float(ref.detach())) <= 2e-6 * abs(float(ref.detach()))


def test_fp16_and_bf16_predictions_are_refused(pvb):
    mask, kpt = _inputs(1, 8, 8, 9, seed=0)
    m, k = torch.from_numpy(mask).to(DEV), torch.from_numpy(kpt).to(DEV)
    for dt in (torch.float16, torch.bfloat16, torch.float64):
        with pytest.raises(RuntimeError, match="float32"):
            pvb.vote_loss(torch.zeros(1, 18, 8, 8, dtype=dt, device=DEV), m, k)
    with pytest.raises(RuntimeError, match=r"\[B,2K,H,W\]"):
        pvb.vote_loss(torch.zeros(1, 16, 8, 8, device=DEV), m, k)


# ---- forward ----------------------------------------------------------------------------------------------------------

def _ulps(a, b):
    ia = np.array([a], np.float32).view(np.int32)[0]
    ib = np.array([b], np.float32).view(np.int32)[0]
    return abs(int(ia) - int(ib))


@pytest.mark.parametrize("B,H,W,seed", [(32, 480, 640, 1), (32, 480, 640, 2), (32, 256, 256, 3), (3, 479, 641, 4)])
def test_forward_against_float64_and_torch(pvb, B, H, W, seed):
    K = 9
    mask_np, kpt_np = _inputs(B, H, W, K, seed=seed)
    mask, kpt = torch.from_numpy(mask_np).to(DEV), torch.from_numpy(kpt_np).to(DEV)
    vertex = pvb.vote_target_batch(mask, kpt)                  # == the restatement (test_target_equals_restatement)
    pred = torch.randn(B, 2 * K, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    got = float(pvb.vote_loss(pred, mask, kpt))
    w = mask[:, None].float()
    x = (pred * w - vertex * w).double()                       # each product and the difference rounded in fp32
    ax = x.abs()
    s64 = float(torch.where(ax < 1, 0.5 * x * x, ax - 0.5).sum())
    wsum = np.float32(float(mask.to(torch.int64).sum()))
    want = np.float32(np.float32(np.float32(s64) / wsum) * (np.float32(1) / np.float32(2 * K)))
    assert _ulps(got, want) <= 1, (got, want)
    ref = float(_reference_loss(pred, mask, vertex))
    rel = abs(got - ref) / abs(ref)
    print(f"[vote_loss] B={B} {H}x{W}: |fused - torch fp32| / torch = {rel:.3e} ({_ulps(got, ref)} ulp)")
    assert rel <= 2e-6


# ---- reproducibility, syncs, threads ----------------------------------------------------------------------------------

def _run_once(pvb, pred_data, mask, kpt, scale=1.0):
    p = pred_data.detach().clone().requires_grad_()
    loss = pvb.vote_loss(p, mask, kpt)
    (loss * scale).backward()
    return loss.detach(), p.grad


def test_bitwise_reproducible_and_sync_free(pvb):
    B, H, W, K = 32, 256, 256, 9
    mask_np, kpt_np = _inputs(B, H, W, K, seed=21)
    mask, kpt = torch.from_numpy(mask_np).to(DEV), torch.from_numpy(kpt_np).to(DEV)
    pred = torch.randn(B, 2 * K, H, W, device=DEV)
    l1, g1 = _run_once(pvb, pred, mask, kpt)
    p = pred.clone().requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = pvb.vote_loss(p, mask, kpt)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _bits_equal(loss.detach(), l1) and _bits_equal(p.grad, g1)
    l2, g2 = _run_once(pvb, pred, mask, kpt)
    assert _bits_equal(l2, l1) and _bits_equal(g2, g1)


def test_side_stream_in_a_thread(pvb):
    B, H, W, K = 4, 96, 128, 9
    mask_np, kpt_np = _inputs(B, H, W, K, seed=31)
    mask, kpt = torch.from_numpy(mask_np).to(DEV), torch.from_numpy(kpt_np).to(DEV)
    pred = torch.randn(B, 2 * K, H, W, device=DEV)
    l1, g1 = _run_once(pvb, pred, mask, kpt, scale=1.5)
    torch.cuda.synchronize()
    out = {}

    def work():
        s = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(s):
            out["r"] = _run_once(pvb, pred, mask, kpt, scale=1.5)
        s.synchronize()

    t = threading.Thread(target=work)
    t.start()
    t.join()
    assert _bits_equal(out["r"][0], l1) and _bits_equal(out["r"][1], g1)


class _Head(torch.nn.Module):
    """A small conv head with PVNet's outputs: 'vertex' (a channel slice) and 'seg'."""

    def __init__(self, K, seed):
        super().__init__()
        torch.manual_seed(seed)
        self.conv = torch.nn.Conv2d(3, 2 * K + 2, 3, padding=1)
        self.K = K

    def forward(self, inp):
        out = self.conv(inp)
        return {'vertex': out[:, :2 * self.K], 'seg': out[:, 2 * self.K:]}


def _batch(B, H, W, K, seed):
    mask_np, kpt_np = _inputs(B, H, W, K, seed=seed)
    g = torch.Generator().manual_seed(seed)
    from clean_pvnet_b200.vote_loss import compact_vertex
    compact = np.stack([compact_vertex(m, k).transpose(2, 0, 1) for m, k in zip(mask_np, kpt_np)])
    return {'inp': torch.randn(B, 3, H, W, generator=g).to(DEV), 'mask': torch.from_numpy(mask_np).to(DEV),
            'vertex': torch.from_numpy(compact).to(DEV), 'meta': {}}, mask_np, kpt_np


def test_network_wrapper_inside_data_parallel(pvb):
    K = 9
    batch, _, _ = _batch(4, 64, 80, K, seed=41)
    head = _Head(K, seed=1).to(DEV)
    w = pvb.NetworkWrapper(head)
    _, loss1, stats1, _ = w(batch)
    loss1.backward()
    g1 = head.conv.weight.grad.clone()
    head.zero_grad(set_to_none=True)
    dp = torch.nn.DataParallel(w, device_ids=[0])
    _, loss2, stats2, _ = dp(batch)
    loss2.mean().backward()
    assert set(stats2) == {'vote_loss', 'seg_loss', 'loss'}
    assert _bits_equal(loss2.reshape(()), loss1.reshape(()))
    assert _bits_equal(stats2['vote_loss'].reshape(()), stats1['vote_loss'].reshape(()))
    assert _bits_equal(head.conv.weight.grad, g1)


def test_one_sgd_step_equals_the_reference_trainer(pvb):
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    K = 9
    batch, mask_np, kpt_np = _batch(4, 64, 80, K, seed=51)
    dense = torch.from_numpy(_restate(mask_np, kpt_np)).to(DEV)

    def step(head, loss_fn):
        opt = torch.optim.SGD(head.parameters(), lr=0.1, momentum=0.9)
        opt.zero_grad()
        loss_fn(head).backward()
        opt.step()
        return [p.detach().clone() for p in head.parameters()]

    def reference(head):                                     # lib/train/trainers/pvnet.py, forward, on the dense field
        output = head(batch['inp'])
        loss = 0
        weight = batch['mask'][:, None].float()
        vote_loss = F.smooth_l1_loss(output['vertex'] * weight, dense * weight, reduction='sum')
        vote_loss = vote_loss / weight.sum() / dense.size(1)
        loss += vote_loss
        loss += torch.nn.CrossEntropyLoss()(output['seg'], batch['mask'].long())
        return loss

    want = step(_Head(K, seed=2).to(DEV), reference)
    got = step(_Head(K, seed=2).to(DEV), lambda head: pvb.NetworkWrapper(head)(batch)[1])
    for a, b in zip(got, want):
        assert _bits_equal(a, b)
