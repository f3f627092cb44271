"""ctypes binding of libssd3d.so (include/ssd3d.h).  There is NO CPU fallback: if the CUDA library is
missing or does not load, importing the operators fails loudly."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SSD3D_LIB") or os.path.join(_HERE, "libssd3d.so")   # override: instrumented builds
_lib = None

c_int, c_long, c_float, c_void_p, c_longlong = ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_void_p, ctypes.c_longlong

# name -> argtypes, exactly the prototypes of include/ssd3d.h
_SIGNATURES = {
    "ssd3d_version": [],
    "ssd3d_fps_needs_temp": [c_int, c_int],
    "ssd3d_farthest_point_sample": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_farthest_point_sample_with_distance": [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_gather_point": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_query_ball_point": [c_int, c_int, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_query_ball_point_dilated": [c_int, c_int, c_int, c_float, c_float, c_int, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p],
    "ssd3d_query_ball_point_multi": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_query_ball_point_workspace": [c_int, c_int],
    "ssd3d_query_ball_point_multi_ws": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_size_t, c_void_p],
    "ssd3d_fill_zero": [c_void_p, c_long, c_void_p],
    "ssd3d_group_point": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_three_nn": [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_three_interpolate": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_calc_square_dist": [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "ssd3d_group_concat": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_void_p],
    "ssd3d_linear_bn_relu": [c_long, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                             c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_rowgroup_max": [c_long, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p],
    "ssd3d_linear_tc": [c_long, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                        c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_linear_tc_hoisted": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int,
                                c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_linear_tc_gather": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                               c_int, c_void_p],
    "ssd3d_hoist_expand_split": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_hoist_expand_split_units": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_linear_tc_units": [c_long, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                              c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_linear_tc_hoisted_units": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int,
                                      c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_split_rows": [c_long, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_group_concat_split": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_int, c_void_p],
    "ssd3d_sa_fused_smem": [c_int, c_int, c_void_p],
    "ssd3d_sa_mlp_fused": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_sa_mlp_fused_hoisted": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                   c_void_p, c_int, c_void_p],
    "ssd3d_gather_point_grad": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_group_point_grad": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_three_interpolate_grad": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_bev_nms": [c_int, c_int, c_void_p, c_void_p, c_float, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "ssd3d_farthest_point_sample_features": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_ffps_supported": [c_int, c_int],
    "ssd3d_farthest_point_sample_ex": [c_int, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_int,
                                       c_int, c_int, c_int, c_int, c_void_p],
    "ssd3d_peer_allgather": [c_void_p, ctypes.c_size_t, c_void_p, c_int, c_int, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t,
                             ctypes.c_size_t, c_void_p, c_void_p, c_void_p],
    "ssd3d_fps_supports_rounds": [c_int, c_int],
    "ssd3d_fps_temp_elems": [c_int, c_int, c_int, c_int],
    "ssd3d_farthest_point_sample_with_distance_ex": [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                                     c_void_p],
    "ssd3d_farthest_point_sample_features_ex": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p,
                                                c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "ssd3d_farthest_point_sample_features_cl": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p,
                                                c_longlong, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "ssd3d_gather_point_ex": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p],
    "ssd3d_concat_rows": [c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p],
    "ssd3d_bn_train_workspace": [c_int],
    "ssd3d_bn_train": [c_long, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_void_p,
                       c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p],
    "ssd3d_split_points": [c_long, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_iota_idx": [c_int, c_int, c_int, c_void_p, c_int, c_void_p],
    "ssd3d_concat_cols": [c_int, c_int, c_int, c_int, c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, c_void_p],
    "ssd3d_vote_translate": [c_long, c_void_p, c_void_p, c_int, c_float, c_float, c_float, c_void_p, c_void_p],
    "ssd3d_decode_dist_anchor_free": [c_long, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                      c_void_p],
    "ssd3d_linear_wgrad_workspace": [c_long, c_int, c_int],
    "ssd3d_linear_wgrad": [c_long, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, ctypes.c_size_t, c_void_p, c_void_p,
                           c_void_p],
    "ssd3d_bn_train_grad_workspace": [c_int],
    "ssd3d_bn_train_grad": [c_long, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                            c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_rowgroup_max_grad": [c_long, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p],
    "ssd3d_group_concat_grad": [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                c_void_p],
    "ssd3d_vote_translate_grad": [c_long, c_void_p, c_int, c_void_p, c_float, c_float, c_float, c_void_p, c_void_p],
    "ssd3d_det_assign": [c_int, c_int, c_int, c_int, c_int] + [c_void_p] * 15,
    "ssd3d_det_loss_workspace": [c_int],
    "ssd3d_det_loss": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int,
                       c_void_p, c_int] + [c_void_p] * 12,
    "ssd3d_det_loss_grad": [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p,
                            c_int, c_void_p, c_int] + [c_void_p] * 11 + [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int,
                                                                         c_void_p, c_int, c_void_p, c_void_p],
    "ssd3d_grad_clip_scale_workspace": [c_long],
    "ssd3d_grad_clip_scale": [c_void_p, c_long, c_float, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_peer_allreduce_resident_ctas": [],
    "ssd3d_peer_allreduce_mean": [c_void_p, ctypes.c_size_t, c_void_p, c_void_p, c_int, c_int, c_int] + [ctypes.c_size_t] * 10 +
                                 [c_void_p, c_void_p],
    "ssd3d_bn_moving_update_ranks": [c_void_p, c_long, c_void_p, c_long, c_int, c_float, c_void_p],
    "ssd3d_adam_step": [c_void_p, c_void_p, c_void_p, c_void_p, c_long, c_void_p, c_float, c_float, c_float, c_int, c_void_p,
                        c_void_p, c_void_p],
    "ssd3d_weight_operands": [c_void_p, c_void_p, c_int, c_long, c_void_p, c_void_p],
    "ssd3d_box_iou": [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_box_iou_matched": [c_long, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "ssd3d_eval_workspace": [c_long],
    "ssd3d_eval_overlaps": [c_int, c_int, c_int] + [c_void_p] * 7,
    "ssd3d_eval_first_pass": [c_int, c_int, c_int] + [c_void_p] * 6 + [c_long] + [c_void_p] * 4,
    "ssd3d_eval_count": [c_int, c_int, c_int] + [c_void_p] * 10,
    "ssd3d_augment_workspace": [c_int, c_int],
    "ssd3d_augment_sem_labels": [c_int, c_int, c_int] + [c_void_p] * 6,
    "ssd3d_augment_boxes": [c_int, c_int] + [c_void_p] * 8,
    "ssd3d_augment_points": [c_int, c_int, c_int] + [c_void_p] * 10,
    "ssd3d_augment_choose": [c_int, c_int] + [c_void_p] * 7,
    "ssd3d_mixup_db_count": [c_int, c_int, c_int] + [c_void_p] * 5,
    "ssd3d_mixup_db_write": [c_int, c_int] + [c_void_p] * 7,
    "ssd3d_mixup_paste_boxes": [c_int, c_int, c_int] + [c_void_p] * 10,
    "ssd3d_mixup_paste_points": [c_int, c_int, c_int] + [c_void_p] * 15,
    "ssd3d_prepare_workspace": [c_int, c_int],
    "ssd3d_prepare_points": [c_int, c_int, c_int] + [c_void_p] * 9,
}

EXPORTS = sorted(list(_SIGNATURES) + ["ssd3d_last_error"])


def lib():
    """Load libssd3d.so (built by `python 3dssd_b200/build.py` / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libssd3d.so is not built (%s missing): run __graft_entry__.build(); "
                               "there is no CPU fallback" % LIB_PATH)
        l = ctypes.CDLL(LIB_PATH)
        for name, argtypes in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.argtypes = argtypes
            fn.restype = ctypes.c_size_t if name in ("ssd3d_sa_fused_smem", "ssd3d_query_ball_point_workspace", "ssd3d_bn_train_workspace",
                                                   "ssd3d_linear_wgrad_workspace", "ssd3d_bn_train_grad_workspace",
                                                   "ssd3d_det_loss_workspace", "ssd3d_grad_clip_scale_workspace",
                                                   "ssd3d_eval_workspace", "ssd3d_augment_workspace",
                                                   "ssd3d_prepare_workspace") else c_int
            if name == "ssd3d_fps_temp_elems":
                fn.restype = c_long
        l.ssd3d_last_error.restype = ctypes.c_char_p
        l.ssd3d_last_error.argtypes = []
        _lib = l
    return _lib


def check(status, op):
    """Map a non-zero C status to the reference's error classes: InvalidArgument -> ValueError,
    anything CUDA -> RuntimeError."""
    if status == 0:
        return
    msg = lib().ssd3d_last_error().decode("utf-8", "replace")
    if status == -1:
        raise ValueError("%s: %s" % (op, msg))
    raise RuntimeError("%s failed (status %d): %s" % (op, status, msg))
