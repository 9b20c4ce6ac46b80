"""ctypes binding of the C ABI in include/delora_b200.h (the "thin torch extension": torch only
supplies device pointers and the current stream).  There is NO fallback: if the shared library
is missing or a GPU is absent the product path raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdelora_b200.so")

c_int, c_float, c_double, c_void_p = ctypes.c_int, ctypes.c_float, ctypes.c_double, ctypes.c_void_p
c_u32, c_i64 = ctypes.c_uint32, ctypes.c_int64


class OdometryDesc(ctypes.Structure):
    """delora_odometry_desc (include/delora_b200.h): the model and buffer sizes of the odometry entry points."""
    _fields_ = [("H", c_int), ("W", c_int), ("hfov0", c_double), ("hfov1", c_double), ("vfov0", c_double),
                ("vfov1", c_double), ("n_stride", c_int), ("max_batch", c_int), ("act", c_int),
                ("layers", c_int * 4), ("resnet_outputs", c_int), ("single_mlp", c_int), ("w_pre", c_int)]


class OdometryTrainParams(ctypes.Structure):
    """delora_odometry_train_params (include/delora_b200.h): Adam, the loss and the normals' settings of a step."""
    _fields_ = [("lr", c_float), ("beta1", c_float), ("beta2", c_float), ("eps", c_float), ("lambda_po2pl", c_float),
                ("loss_flags", c_u32), ("nb_h", c_int), ("nb_w", c_int), ("epsilon_range", c_float),
                ("min_neighbors", c_int)]


class OdometryResidualParams(ctypes.Structure):
    """delora_odometry_residual_params (include/delora_b200.h): the loss and the normals' settings of the per-frame ICP
    residual of delora_odometry_streams_push_residual."""
    _fields_ = [("lambda_po2pl", c_float), ("loss_flags", c_u32), ("nb_h", c_int), ("nb_w", c_int),
                ("epsilon_range", c_float), ("min_neighbors", c_int)]


GRAD_ALLREDUCE_MAX_WORLD = 16       # DELORA_GRAD_ALLREDUCE_MAX_WORLD
TRAIN_GROUP_BUCKETS = 5             # DELORA_TRAIN_GROUP_BUCKETS


class OdometryTrainGroup(ctypes.Structure):
    """delora_odometry_train_group (include/delora_b200.h): one rank's view of a data-parallel training group."""
    _fields_ = [("rank", ctypes.c_int32), ("world", ctypes.c_int32),
                ("peer_ws", ctypes.c_uint64 * GRAD_ALLREDUCE_MAX_WORLD),
                ("peer_flags", ctypes.c_uint64 * GRAD_ALLREDUCE_MAX_WORLD), ("multicast", ctypes.c_uint64),
                ("n_ctas", ctypes.c_int32), ("n_threads", ctypes.c_int32), ("status", c_void_p),
                ("side_stream", c_void_p), ("fork_events", c_void_p * TRAIN_GROUP_BUCKETS), ("join_event", c_void_p)]


class WsSection(ctypes.Structure):
    """delora_ws_section (include/delora_b200.h): one section of an odometry workspace's layout."""
    _fields_ = [("offset", c_i64), ("bytes", c_i64), ("role", ctypes.c_int32), ("geometry", ctypes.c_int32),
                ("flags", ctypes.c_int32), ("name", ctypes.c_char * 44)]


# workspace kinds, section roles and flags of delora_odometry_workspace_sections (DELORA_WS_* in include/delora_b200.h)
WS_KINDS = ("pairs", "streams", "streams_residual", "streams_info", "streams_normalized", "streams_pre",
            "streams_pre_info", "train", "train_geometries", "adapt", "adapt_group", "adapt_info", "adapt_geometries",
            "adapt_geometries_info")
WS_ROLES = ("weights", "state", "scratch", "output")
WS_SUBRANGE, WS_SHARED = 1, 2

c_desc_p = ctypes.POINTER(OdometryDesc)
c_train_p = ctypes.POINTER(OdometryTrainParams)
c_residual_p = ctypes.POINTER(OdometryResidualParams)
c_group_p = ctypes.POINTER(OdometryTrainGroup)

# name -> (restype, argtypes); every symbol declared in include/delora_b200.h
SIGNATURES = {
    "delora_abi_version": (c_int, []),
    "delora_last_error": (ctypes.c_char_p, []),
    "delora_project_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double,
                                   c_double, c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_project_uv": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double,
                                  c_double, c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_sort_scratch_bytes": (c_i64, [c_int, c_int]),
    "delora_sort_by_range": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_normals_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p,
                                   c_void_p, c_void_p, c_void_p]),
    "delora_project_normals_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double,
                                           c_double, c_double, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                           c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_project_points_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double,
                                          c_double, c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p]),
    "delora_scan_blocks": (c_int, [c_int]),
    "delora_lists_from_images": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_grid_build": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_double, c_double,
                                  c_double, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_grids_from_projection": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                             c_void_p, c_void_p, c_void_p]),
    "delora_project_grids_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_double, c_double, c_double,
                                         c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_pack_lists": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_icp_partial_rows": (c_int, [c_int]),
    "delora_icp_scratch_floats": (c_i64, [c_int, c_int]),
    "delora_icp_stats": (c_int, [c_void_p, c_int]),
    "delora_icp_dense_fwd_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_double, c_double, c_double, c_double, c_float, c_u32, c_void_p,
                                         c_void_p, c_void_p, c_void_p]),
    "delora_icp_information_scratch_floats": (c_i64, [c_int, c_int, c_int]),
    "delora_icp_dense_information": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                             c_double, c_double, c_double, c_double, c_float, c_u32, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_icp_dense_information_scaled": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                    c_int, c_double, c_double, c_double, c_double, c_float, c_u32,
                                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                    c_void_p]),
    "delora_icp_fwd_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_int, c_int, c_int, c_int, c_double, c_double, c_double, c_double, c_float,
                                   c_u32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_icp_point_grads": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p]),
    "delora_conv2d_fprop_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "delora_conv2d_dgrad_eligible": (c_int, [c_int, c_int, c_int, c_int, c_int]),
    "delora_conv2d_dgrad_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "delora_conv2d_wgrad_scratch_floats": (c_i64, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "delora_conv2d_wgrad_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_int, c_int, c_void_p]),
    "delora_zero_upsample_nhwc_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                               c_void_p]),
    "delora_images_to_nhwc_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "delora_maxpool_w_nhwc_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "delora_maxpool_w_idx_nhwc_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                               c_void_p]),
    "delora_maxpool_w_bwd_nhwc_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                               c_int, c_void_p]),
    "delora_avgpool_nhwc_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "delora_avgpool_bwd_nhwc_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "delora_conv_weight_prep_bf16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_conv_weight_prep_multi": (c_int, [c_void_p, c_int, c_void_p]),
    "delora_images_to_nhwc16_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "delora_stem_weight_prep_bf16": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "delora_stem_fprop_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "delora_stem_wgrad_scratch_floats": (c_i64, [c_int, c_int, c_int]),
    "delora_stem_wgrad_bf16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "delora_nhwc_to_nchw_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "delora_quat_to_T": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "delora_quat_to_T_bwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_grad_allreduce_flag_words": (c_int, []),
    "delora_grad_allreduce_f32": (c_int, [c_void_p, c_void_p, ctypes.c_uint64, c_int, c_int, ctypes.c_longlong,
                                          ctypes.c_longlong, c_float, c_u32, c_int, c_int, c_void_p, c_void_p]),
    "delora_trunk_weight_bytes": (c_i64, [c_void_p, c_int]),
    "delora_trunk_prep_weights": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_trunk_activation_bytes": (c_i64, [c_void_p, c_int, c_int, c_int, c_int]),
    "delora_trunk_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    "delora_trunk_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_int, c_void_p]),
    "delora_trunk_forward_dropout": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_trunk_backward_dropout": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                              c_void_p, c_int, c_void_p, c_void_p]),
    "delora_odometry_file_objective": (c_int, [c_void_p, c_void_p, c_void_p]),
    "delora_odometry_weight_floats": (c_i64, [c_desc_p]),
    "delora_odometry_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_init": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_load_weights": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_pairs": (c_int, [c_desc_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_push": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_normalization_factors": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "delora_odometry_pairs_normalized": (c_int, [c_desc_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                                 c_void_p, c_void_p]),
    "delora_odometry_streams_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_init": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_streams_load_weights": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p]),
    "delora_odometry_streams_reset": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_residual_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_residual_init": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_residual": (c_int, [c_desc_p, c_residual_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                      c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_info_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_info_init": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_info": (c_int, [c_desc_p, c_residual_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_normalized_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_normalized_init": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_normalized": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                        c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_pre_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_pre_init": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_pre": (c_int, [c_desc_p, c_residual_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_pre_info_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_pre_info_init": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_pre_info": (c_int, [c_desc_p, c_residual_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_train_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_train_init": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_train_step": (c_int, [c_desc_p, c_train_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p]),
    "delora_odometry_train_step_group": (c_int, [c_desc_p, c_train_p, c_group_p, c_void_p, c_void_p, c_int, c_void_p,
                                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_train_grad_offset": (c_i64, [c_desc_p]),
    "delora_odometry_train_group_buckets": (c_int, [c_desc_p, c_void_p, c_void_p]),
    "delora_odometry_train_geometries_workspace_bytes": (c_i64, [c_desc_p, c_int]),
    "delora_odometry_train_geometries_init": (c_int, [c_desc_p, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_train_use_geometry": (c_int, [c_desc_p, c_int, c_int, c_void_p, c_void_p]),
    "delora_odometry_train_eval": (c_int, [c_desc_p, c_train_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p]),
    "delora_odometry_train_weights": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_train_get_state": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_train_set_state": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_adapt_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_adapt_init": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_adapt": (c_int, [c_desc_p, c_train_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                                   c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_adapt_reset": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_adapt_group_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_adapt_group_init": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_adapt_group": (c_int, [c_desc_p, c_train_p, c_group_p, c_int, c_void_p, c_void_p,
                                                         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_adapt_info_workspace_bytes": (c_i64, [c_desc_p]),
    "delora_odometry_streams_adapt_info_init": (c_int, [c_desc_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_adapt_info": (c_int, [c_desc_p, c_train_p, c_int, c_void_p, c_void_p, c_void_p,
                                                        c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_adapt_group_info": (c_int, [c_desc_p, c_train_p, c_group_p, c_int, c_void_p,
                                                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                              c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_adapt_geometries_workspace_bytes": (c_i64, [c_desc_p, c_int]),
    "delora_odometry_streams_adapt_geometries_init": (c_int, [c_desc_p, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_push_adapt_geometries": (c_int, [c_desc_p, c_int, c_train_p, c_int, c_void_p, c_void_p,
                                                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                              c_void_p]),
    "delora_odometry_streams_adapt_geometries_reset": (c_int, [c_desc_p, c_int, c_void_p, c_void_p, c_void_p]),
    "delora_odometry_streams_adapt_geometries_info_workspace_bytes": (c_i64, [c_desc_p, c_int]),
    "delora_odometry_streams_push_adapt_geometries_info": (c_int, [c_desc_p, c_int, c_train_p, c_int, c_void_p,
                                                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                                   c_void_p, c_void_p, c_void_p]),
    "delora_odometry_workspace_sections": (c_int, [c_int, c_desc_p, c_int, c_void_p, c_int]),
    "delora_odometry_train_set_dropout_seed":(c_int, [c_desc_p, ctypes.c_uint64, c_void_p, c_void_p]),
    "delora_dropout_keep_mask": (c_int, [ctypes.c_uint64, c_i64, c_int, c_i64, c_void_p, c_void_p]),
}

ABI_VERSION = 3
# model_flags bits of the .dlw / .dlt header (DELORA_MODEL_* in include/delora_b200.h)
MODEL_NORMALIZATION_SCALING = 1
MODEL_DROPOUT = 2
# the loss_flags bits a .dlw / .dlt header's objective_flags holds (DELORA_LOSS_* / DELORA_NORMAL_LINEAR)
LOSS_PO2PO, LOSS_PO2PL, LOSS_PL2PL, NORMAL_LINEAR, LOSS_PO2PO_ALONE = 1, 2, 4, 8, 4096
_lib = None


def lib():
    """Load libdelora_b200.so (built by `python -m delora_b200.build` / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"delora_b200: {LIB_PATH} is missing. Build it with `python delora_b200/build.py` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    handle = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(handle, name)          # AttributeError if the library does not export it
        fn.restype = restype
        fn.argtypes = argtypes
    if handle.delora_abi_version() != ABI_VERSION:
        raise RuntimeError("delora_b200: ABI version mismatch between _lib.py and libdelora_b200.so")
    _lib = handle
    return _lib


def check(status, what):
    if status != 0:
        msg = lib().delora_last_error()
        raise RuntimeError(f"{what} failed ({status}): {msg.decode() if msg else ''}")
