"""CPU tests of the evaluator metrics' C ABI (pvb_pose_metrics, pvb_mask_iou) and Python surface (clean_pvnet_b200.metrics):
argument validation happens before any CUDA call, so no device is needed."""
import ctypes

import numpy as np
import pytest
import torch


def _buf():
    buf = ctypes.create_string_buffer(4096)
    return buf, ctypes.addressof(buf)


def test_pose_metrics_validation(pvb):
    lib = pvb._lib.load()
    INV, WS, OK = pvb._lib.PVB_ERR_INVALID, pvb._lib.PVB_ERR_WORKSPACE, pvb._lib.PVB_OK
    _keep, p = _buf()
    pm = lib.pvb_pose_metrics
    # model, pose_pred, pose_gt, K, k_stride, proj2d, trans_cm, angle_deg, n, pn, workspace, bytes, stream
    assert pm(p, p, p, p, 0, p, p, p, -1, 10, p, 4096, None) == INV
    assert pm(p, p, p, p, 0, p, p, p, 1, -10, p, 4096, None) == INV
    assert b"negative size" in lib.pvb_last_error()
    for i in range(8):
        if i == 4:
            continue                                    # k_stride, not a pointer
        args = [p, p, p, p, 0, p, p, p]
        args[i] = None
        assert pm(*args, 2, 10, p, 4096, None) == INV, i
        assert b"NULL" in lib.pvb_last_error()
    assert pm(p, p, p, p, -9, p, p, p, 2, 10, p, 4096, None) == INV
    assert b"stride" in lib.pvb_last_error()
    # n == 0 is a no-op whatever the pointers; pn == 0 needs no model
    assert pm(None, None, None, None, 0, None, None, None, 0, 10, None, 0, None) == OK
    assert pm(None, None, None, None, -5, None, None, None, 0, 0, None, 0, None) == OK
    need = lib.pvb_pose_metrics_workspace_bytes(4, 5000)
    assert need == 4 * 3 * 8                            # one partial sum per pair and chunk of 2048 points
    assert pm(p, p, p, p, 0, p, p, p, 4, 5000, None, 0, None) == WS
    assert pm(p, p, p, p, 0, p, p, p, 4, 5000, p, need - 1, None) == WS
    assert b"workspace" in lib.pvb_last_error()


def test_pose_metrics_workspace_sizing(pvb):
    ws = pvb._lib.load().pvb_pose_metrics_workspace_bytes
    assert ws(1, 1) == 8 and ws(1, 2048) == 8 and ws(1, 2049) == 16
    assert ws(300, 20000) == 300 * 10 * 8
    assert ws(7, 0) == 0 and ws(0, 1000) == 0 and ws(-1, 1000) == 0 and ws(3, -1) == 0


def test_mask_iou_validation(pvb):
    lib = pvb._lib.load()
    L = pvb._lib
    INV, OK = L.PVB_ERR_INVALID, L.PVB_OK
    _keep, p = _buf()
    s = (ctypes.c_int64 * 3)(307200, 640, 1)
    mi = lib.pvb_mask_iou
    I64, U8 = L.PVB_MASK_I64, L.PVB_MASK_U8
    # pred, pred_dtype, pred_stride, gt, gt_dtype, gt_stride, inter, uni, B, H, W, stream
    for B, H, W in ((-1, 480, 640), (1, -480, 640), (1, 480, -640)):
        assert mi(p, I64, s, p, U8, s, p, p, B, H, W, None) == INV
    for bad in (L.PVB_MASK_F32, L.PVB_MASK_F64, 7, -1):
        assert mi(p, bad, s, p, U8, s, p, p, 1, 480, 640, None) == INV
        assert mi(p, I64, s, p, bad, s, p, p, 1, 480, 640, None) == INV
        assert b"dtype" in lib.pvb_last_error()
    assert mi(p, I64, None, p, U8, s, p, p, 1, 480, 640, None) == INV
    assert mi(p, I64, s, p, U8, None, p, p, 1, 480, 640, None) == INV
    assert b"stride array" in lib.pvb_last_error()
    for i in (0, 3, 6, 7):
        args = [p, I64, s, p, U8, s, p, p]
        args[i] = None
        assert mi(*args, 1, 480, 640, None) == INV, i
        assert b"NULL tensor" in lib.pvb_last_error()
    neg = (ctypes.c_int64 * 3)(307200, -640, 1)
    assert mi(p, I64, neg, p, U8, s, p, p, 1, 480, 640, None) == INV
    assert mi(p, I64, s, p, U8, neg, p, p, 1, 480, 640, None) == INV
    assert mi(p, I64, s, p, U8, s, p, p, 1, 65536, 32768, None) == INV      # H*W = 2^31
    assert b"too large" in lib.pvb_last_error()
    # B == 0 is a no-op, even with NULL tensors and stride arrays
    assert mi(None, I64, None, None, U8, None, None, None, 0, 480, 640, None) == OK


def test_python_surface_rejects_bad_inputs(pvb):
    m, pose, K = np.zeros((10, 3)), np.zeros((4, 3, 4)), np.eye(3)
    with pytest.raises(RuntimeError, match="model"):
        pvb.pose_metrics_batch(np.zeros((10, 2)), pose, pose, K)
    with pytest.raises(RuntimeError, match=r"\[n,3,4\]"):
        pvb.pose_metrics_batch(m, np.zeros((4, 4, 4)), np.zeros((4, 4, 4)), K)
    with pytest.raises(RuntimeError, match=r"\[n,3,4\]"):
        pvb.pose_metrics_batch(m, pose, pose[:3], K)
    with pytest.raises(RuntimeError, match="K must be"):
        pvb.pose_metrics_batch(m, pose, pose, np.zeros((3, 3, 3)))
    with pytest.raises(RuntimeError, match="K must be"):
        pvb.linemod_scores(m, 0.1, pose, pose, np.zeros((4, 3)))
    with pytest.raises(RuntimeError, match="or neither"):
        pvb.linemod_scores(m, 0.1, pose, pose, K, mask_pred=torch.zeros(4, 8, 8, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        pvb.mask_iou_batch(torch.zeros(1, 8, 8, dtype=torch.int64), torch.zeros(1, 8, 8, dtype=torch.uint8))
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        pvb.mask_iou_batch(np.zeros((1, 8, 8), np.int64), np.zeros((1, 8, 8), np.uint8))
    assert pvb.metrics.pose_metrics_batch is pvb.pose_metrics_batch
    assert pvb.metrics.linemod_scores is pvb.linemod_scores
