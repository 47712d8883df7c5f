"""ctypes binding of libpvnet_vote_b200.so (the C ABI of include/pvnet_vote_b200.h).

The library is hand-written sm_90a (H100) CUDA; there is deliberately no CPU or PyTorch
fallback -- if the shared object is missing, importing the ops raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpvnet_vote_b200.so")

PVB_OK, PVB_ERR_INVALID, PVB_ERR_CUDA, PVB_ERR_WORKSPACE, PVB_ERR_CAPACITY, PVB_ERR_TIMEOUT = range(6)
PVB_HOST_STAGE_VERTEX, PVB_HOST_INPLACE_MASK = 2, 4
PVB_IPC_HANDLE_BYTES = 64
(PVB_MASK_U8, PVB_MASK_I8, PVB_MASK_I16, PVB_MASK_I32, PVB_MASK_I64, PVB_MASK_F32, PVB_MASK_F64) = range(7)
PVB_SELECT_BYTE, PVB_SELECT_EQ1 = 0, 1
PVB_CROP_MASK_TO_BOX, PVB_CROP_CENTER_F64 = 1, 2
(PVB_PNP_OK, PVB_PNP_ITERATION_LIMIT, PVB_PNP_TOO_FEW_POINTS, PVB_PNP_PLANAR, PVB_PNP_DEGENERATE) = range(5)
PVB_DCN_F16, PVB_DCN_BF16 = 1, 2


class PvbDesc(ctypes.Structure):
    _fields_ = [
        ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32), ("K", ctypes.c_int32),
        ("hn", ctypes.c_int32),
        ("inlier_thresh", ctypes.c_float),
        ("min_num", ctypes.c_int32), ("max_num", ctypes.c_int32),
        ("mask_dtype", ctypes.c_int32), ("select_mode", ctypes.c_int32),
        ("mask_stride", ctypes.c_int64 * 3),
        ("vertex_stride", ctypes.c_int64 * 5),
        ("capacity", ctypes.c_int32), ("img_base", ctypes.c_int32),
        ("seed", ctypes.c_uint64),
        ("rng_tag_idx", ctypes.c_int32), ("rng_tag_sel", ctypes.c_int32),
    ]


class PvbLayout(ctypes.Structure):
    _fields_ = [(n, ctypes.c_size_t) for n in
                ("total", "status", "fgsum", "nz", "tn", "state", "bits", "ticket", "blocktot", "xy", "dirs", "hyp",
                 "counts", "win", "refit_partial", "refit_ticket", "prune_cells", "prune_key", "prune_list", "prune_len")] + [
                    ("nwords", ctypes.c_int32), ("nblocks", ctypes.c_int32), ("capacity", ctypes.c_int32),
                    ("refit_splits", ctypes.c_int32), ("prune_ncells", ctypes.c_int32)]


class PvbPnpOptions(ctypes.Structure):
    """== struct pvb_pnp_options (include/pvnet_vote_b200.h)"""
    _fields_ = [("max_num_iterations", ctypes.c_int32), ("reserved", ctypes.c_int32),
                ("function_tolerance", ctypes.c_double), ("gradient_tolerance", ctypes.c_double),
                ("parameter_tolerance", ctypes.c_double)]


class PvbDcnDesc(ctypes.Structure):
    """== struct pvb_dcn_desc (include/pvnet_vote_b200.h)"""
    _fields_ = [(n, ctypes.c_int32) for n in ("B", "C", "H", "W", "C_out", "kh", "kw", "stride_h", "stride_w", "pad_h",
                                             "pad_w", "dilation_h", "dilation_w", "deformable_groups")]


class PvbDcnPoolDesc(ctypes.Structure):
    """== struct pvb_dcn_pool_desc (include/pvnet_vote_b200.h)"""
    _fields_ = [(n, ctypes.c_int32) for n in ("B", "C", "H", "W", "n_roi", "output_dim", "pooled_size", "part_size",
                                             "sample_per_part", "group_size", "num_classes", "no_trans")] + [
        ("spatial_scale", ctypes.c_float), ("trans_std", ctypes.c_float)]


# every symbol include/pvnet_vote_b200.h declares: name -> (restype, argtypes)
_vp, _i32, _sz, _f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_size_t, ctypes.c_float
_dp, _lp = ctypes.POINTER(PvbDesc), ctypes.POINTER(PvbLayout)
SIGNATURES = {
    "pvb_version": (ctypes.c_int, []),
    "pvb_last_error": (ctypes.c_char_p, []),
    "pvb_workspace_bytes": (_sz, [_dp]),
    "pvb_workspace_layout": (ctypes.c_int, [_dp, _lp]),
    "pvb_ransac_voting_v3": (ctypes.c_int, [_dp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "pvb_decode_v3": (ctypes.c_int, [_dp, _vp, _i32, ctypes.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "pvb_estimate_voting_distribution": (ctypes.c_int, [_dp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "pvb_uncertainty_weights": (ctypes.c_int, [_vp, _vp, _i32, _vp]),
    "pvb_uncertainty_pnp": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, ctypes.c_int64, ctypes.c_int64,
                                           ctypes.c_void_p, _vp]),
    "pvb_uncertainty_pnp_from_votes": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32,
                                                      ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p, _vp]),
    "pvb_uncertainty_pnp_init": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, ctypes.c_int64, ctypes.c_int64, _vp]),
    "pvb_pnp_iterative": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, ctypes.c_int64, ctypes.c_int64, _vp]),
    "pvb_nearest_point_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "pvb_nearest_point_idx": (ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "pvb_add_metric_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "pvb_add_metric": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _sz, _vp]),
    "pvb_pose_metrics_workspace_bytes": (_sz, [_i32, _i32]),
    "pvb_pose_metrics": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_int64, _vp, _vp, _vp, _i32, _i32, _vp, _sz, _vp]),
    "pvb_mask_iou": (ctypes.c_int, [_vp, _i32, ctypes.POINTER(ctypes.c_int64), _vp, _i32, ctypes.POINTER(ctypes.c_int64),
                                    _vp, _vp, _i32, _i32, _i32, _vp]),
    "pvb_render_depth_workspace_bytes": (_sz, [_i32, _i32]),
    "pvb_render_depth": (ctypes.c_int, [_vp, _i32, _vp, _i32, _vp, _i32, _vp, ctypes.c_int64, _vp, _i32, _i32,
                                        ctypes.c_double, ctypes.c_double, _vp, _sz, _vp]),
    "pvb_vsd_workspace_bytes": (_sz, [_i32]),
    "pvb_vsd": (ctypes.c_int, [_vp, _i32, _vp, _i32, _i32, _vp, _i32, _i32, _vp, _i32, _vp, ctypes.c_int64, _i32, _i32,
                               ctypes.c_double, ctypes.c_double, _vp, _vp, _sz, _vp]),
    "pvb_instance_masks_workspace_bytes": (_sz, [_i32, _i32]),
    "pvb_instance_masks": (ctypes.c_int, [_vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _sz,
                                          _vp]),
    "pvb_fps_workspace_bytes": (_sz, [_i32, _i32]),
    "pvb_farthest_point_sampling": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _vp, _sz, _vp]),
    "pvb_crop_inputs": (ctypes.c_int, [_vp, _i32, _i32, _i32, ctypes.POINTER(ctypes.c_int64), _vp, _vp, _i32, _i32, _i32,
                                       ctypes.c_double, ctypes.c_double, _i32, ctypes.POINTER(ctypes.c_float),
                                       ctypes.POINTER(ctypes.c_float), _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pvb_uncrop_keypoints": (ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "pvb_warp_affine_linear": (ctypes.c_int, [_vp, _i32, _i32, _i32, _i32, ctypes.POINTER(ctypes.c_int64), _vp, _vp, _i32,
                                              _i32, _i32, _vp, _vp]),
    "pvb_vote_target":(ctypes.c_int, [_vp, _i32, ctypes.POINTER(ctypes.c_int64), _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "pvb_vote_loss_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "pvb_vote_loss_forward": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int64), _vp, _i32, ctypes.POINTER(ctypes.c_int64),
                                             _vp, _vp, _i32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "pvb_vote_loss_backward": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int64), _vp, _i32, ctypes.POINTER(ctypes.c_int64),
                                              _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "pvb_ct_target": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "pvb_ct_loss_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "pvb_ct_loss_forward": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int64), _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32,
                                           _i32, _i32, _vp, _sz, _vp]),
    "pvb_ct_loss_backward": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int64), _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32,
                                            _i32, _i32, _i32, _vp, _sz, _vp]),
    "pvb_ct_decode_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32]),
    "pvb_ct_decode": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_int64), _vp, ctypes.POINTER(ctypes.c_int64), _i32, _i32,
                                     _i32, _i32, _i32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "pvb_dcn_forward": (ctypes.c_int, [ctypes.POINTER(PvbDcnDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pvb_dcn_forward_half": (ctypes.c_int, [ctypes.POINTER(PvbDcnDesc), _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pvb_dcn_forward_half_nhwc": (ctypes.c_int, [ctypes.POINTER(PvbDcnDesc), _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pvb_dcn_backward_workspace_bytes": (_sz, [ctypes.POINTER(PvbDcnDesc), _i32]),
    "pvb_dcn_backward": (ctypes.c_int, [ctypes.POINTER(PvbDcnDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _i32, _vp, _sz, _vp]),
    "pvb_dcn_forward_tf32": (ctypes.c_int, [ctypes.POINTER(PvbDcnDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pvb_dcn_backward_tf32": (ctypes.c_int, [ctypes.POINTER(PvbDcnDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                             _vp, _i32, _vp, _sz, _vp]),
    "pvb_dcn_pool_forward": (ctypes.c_int, [ctypes.POINTER(PvbDcnPoolDesc), _vp, _vp, _vp, _vp, _vp, _vp]),
    "pvb_dcn_pool_backward": (ctypes.c_int, [ctypes.POINTER(PvbDcnPoolDesc), _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "pvb_read_status": (ctypes.c_int, [_dp, _vp, _vp]),
    "pvb_host_scratch_bytes": (_sz, [_dp, _i32]),
    "pvb_ransac_voting_v3_host": (ctypes.c_int, [_dp, _vp, _vp, _vp, _i32, ctypes.c_uint32, _vp, _sz, _vp]),
    "pvb_exchange_create": (ctypes.c_int, [_i32, _i32, _i32, _sz, ctypes.POINTER(ctypes.c_void_p)]),
    "pvb_exchange_bytes_per_rank": (_sz, [_vp]),
    "pvb_exchange_base": (ctypes.c_void_p, [_vp]),
    "pvb_exchange_get_handle": (ctypes.c_int, [_vp, _vp]),
    "pvb_exchange_connect": (ctypes.c_int, [_vp, _vp]),
    "pvb_exchange_connect_ptrs": (ctypes.c_int, [_vp, ctypes.POINTER(ctypes.c_void_p)]),
    "pvb_ransac_voting_v3_push": (ctypes.c_int, [_dp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, ctypes.c_uint64, _vp]),
    "pvb_ransac_voting_v3_all_counts": (ctypes.c_int, [_dp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, ctypes.c_uint64, _vp]),
    "pvb_estimate_voting_distribution_push": (ctypes.c_int, [_dp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, ctypes.c_uint64, _vp]),
    "pvb_exchange_wait": (ctypes.c_int, [_vp, ctypes.c_uint64, _vp, _vp, ctypes.c_double, _vp]),
    "pvb_exchange_status": (ctypes.c_int, [_vp, _vp]),
    "pvb_exchange_destroy": (ctypes.c_int, [_vp]),
    "pvb_profile_enable": (ctypes.c_int, [_i32]),
    "pvb_profile_reset": (ctypes.c_int, []),
    "pvb_set_tuning": (ctypes.c_int, [_i32, _i32]),
    "pvb_set_pass1_stats": (ctypes.c_int, [_vp]),
    "pvb_set_group_tuning": (ctypes.c_int, [_i32, _i32]),
    "pvb_profile_read": (ctypes.c_int, [ctypes.POINTER(ctypes.c_double), _i32]),
    "pvb_generate_hypothesis": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "pvb_voting_for_hypothesis": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _f, _vp]),
    "pvb_generate_hypothesis_vanishing_point": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "pvb_voting_for_hypothesis_vanishing_point": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _f, _vp]),
    "pvb_vote_count": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _f, _vp, _sz, _vp]),
    "pvb_vote_count_workspace_bytes": (_sz, [_i32, _i32, _i32]),
}

_LIB = None


def load():
    """Loads the CUDA library; raises (never falls back) when it has not been built."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python clean_pvnet_b200/build.py` "
                "(or __graft_entry__.build()). There is no CPU/PyTorch fallback for this op.")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
        if os.environ.get("PVB_VOTE_VARIANT"):     # tooling: A/B the vote-kernel launch shapes
            check(lib.pvb_set_tuning(0, int(os.environ["PVB_VOTE_VARIANT"])))
    return _LIB


def check(rc):
    if rc != PVB_OK:
        msg = load().pvb_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"pvnet_vote_b200 error {rc}: {msg}")
