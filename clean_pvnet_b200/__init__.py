"""clean_pvnet_b200 -- H100-native RANSAC voting layer (drop-in for clean-pvnet's lib/csrc/ransac_voting).

Public surface (same names/signatures as the reference):
    ransac_voting_gpu.ransac_voting_layer / ransac_voting_layer_v3 / estimate_voting_distribution_with_mean
    ransac_voting.generate_hypothesis / voting_for_hypothesis / *_vanishing_point   (the pybind twins)
    un_pnp.uncertainty_pnp / uncertainty_pnp_v2 (twins of lib/csrc/uncertainty_pnp/un_pnp_utils.py), uncertainty_pnp_batch,
    uncertainty_pnp_from_votes (the evaluator's whole un_pnp tail in one launch)
    parallel.ShardedVotingLayer (images sharded over the GPUs of one box, results exchanged over NVLink peer memory)
    nn.find_nearest_point_idx (twin of lib/csrc/nn/nn_utils.py), nearest_point_idx, add_metric_batch (the evaluators'
    ADD / ADD-S distance for n pose pairs), install_nn_as_reference_module
    metrics.pose_metrics_batch (projection_2d / cm_degree_5 distances), mask_iou_batch, linemod_scores (the evaluator's four
    per-image flags for a batch)
    pose.pnp (twin of lib/utils/pvnet/pvnet_pose_utils.py's cv2.solvePnP ITERATIVE step), pnp_batch (n problems, one launch:
    the pose step of the default un_pnp=False path)
    vote_loss.vote_loss (the trainer's vote loss and its gradient from the mask and the keypoints), vote_target_batch (twin
    of lib/utils/pvnet/pvnet_data_utils.py's compute_vertex), NetworkWrapper (twin of lib/train/trainers/pvnet.py),
    install_vote_loss_as_reference
"""
from . import _lib  # noqa: F401
from . import nn  # noqa: F401
from .nn import find_nearest_point_idx, nearest_point_idx, add_metric_batch, install_nn_as_reference_module  # noqa: F401
from . import metrics  # noqa: F401
from .metrics import pose_metrics_batch, mask_iou_batch, linemod_scores  # noqa: F401
from . import ransac_voting  # noqa: F401
from . import ransac_voting_gpu  # noqa: F401
from . import decode  # noqa: F401
from . import parallel  # noqa: F401
from .decode import decode_keypoint, uncertainty_pnp_weights  # noqa: F401
from . import uncertainty_pnp as un_pnp  # noqa: F401
from .uncertainty_pnp import uncertainty_pnp_batch, p3p_init_batch, uncertainty_pnp_from_votes  # noqa: F401
from . import pose  # noqa: F401
from .pose import pnp_batch  # noqa: F401
from .vote_loss import vote_loss, vote_target_batch, NetworkWrapper, install_vote_loss_as_reference  # noqa: F401
from .ransac_voting_gpu import (  # noqa: F401
    estimate_voting_distribution_with_mean,
    ransac_voting_layer,
    ransac_voting_layer_v3,
    ransac_voting_layer_v3_host,
    install_as_reference_module,
)

__all__ = [
    "ransac_voting_layer", "ransac_voting_layer_v3", "estimate_voting_distribution_with_mean",
    "ransac_voting_layer_v3_host", "install_as_reference_module", "ransac_voting", "ransac_voting_gpu",
    "decode_keypoint", "uncertainty_pnp_weights", "un_pnp", "uncertainty_pnp_batch", "p3p_init_batch",
    "uncertainty_pnp_from_votes", "pose", "pnp_batch", "parallel",
    "nn", "find_nearest_point_idx", "nearest_point_idx", "add_metric_batch", "install_nn_as_reference_module",
    "metrics", "pose_metrics_batch", "mask_iou_batch", "linemod_scores",
    "vote_loss", "vote_target_batch", "NetworkWrapper", "install_vote_loss_as_reference",
]
