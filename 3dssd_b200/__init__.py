"""3dssd_b200 -- H100 (sm_90a) set-abstraction operators behind the tf_ops / layers_util surface of
dvlab-research/3DSSD.  Import with importlib.import_module("3dssd_b200") or through the `ssd3d_b200` alias.
"""
from . import augment, config, dist, evaluation, head, kitti_io, layers_util, loss, mixup, params, prepare, solver, tf_ops  # noqa: F401
from ._lib import EXPORTS, LIB_PATH, lib  # noqa: F401
from .backbone import SABackbone, train_forward  # noqa: F401
from .head import DetectionHead  # noqa: F401
from .loss import assign_targets, detection_loss  # noqa: F401
from .params import TrainableParams  # noqa: F401
from .layers_util import (pointnet_fp_module, pointnet_sa_module, pointnet_sa_module_msg,  # noqa: F401
                          vote_layer)
from .tf_ops import (bev_nms, calc_square_dist, farthest_point_sample, farthest_point_sample_with_distance,  # noqa: F401
                     farthest_point_sample_features, ffps_supported,
                     furthest_point_sample, gather_point, gather_point_grad, group_point_grad, three_interpolate_grad, group_concat, group_concat_split, group_point, linear_bn_relu,
                     linear_tc, linear_tc_gather, linear_tc_hoisted, sa_mlp_fused, sa_mlp_fused_hoisted, split_rows,
                     query_ball_point, query_ball_point_dilated, query_ball_point_multi, three_interpolate,
                     three_nn)

__version__ = "0.1.0"
