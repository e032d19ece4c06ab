"""ctypes binding of libcasmvs.so (C ABI declared in include/casmvs.h).

There is deliberately no fallback: if the shared library is missing or the
device is not a H100 (sm_90a) GPU the import / call fails loudly.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_uint64, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libcasmvs.so")

NCHW, NHWC = 0, 1
ROUND_TF32 = 256
KEEP_FP32_OUT = 256      # OR-ed into conv3d precision
BLOCKED = 512            # OR-ed into costreg precision / warp_cost_ladder round_tf32
FUSED_TAIL = 1024        # OR-ed into costreg precision: conv11 + prob in one kernel, u11 not kept
INVERSE_DEPTH = 2048     # OR-ed into regress input_is_prob / regress_bwd dv_is_vector / warp_cost_ladder round_tf32
FP32, TF32 = 0, 1
CONV, CONV_TRANSPOSE, CONV_PLANAR = 0, 1, 2
PRECISIONS = {"fp32": FP32, "tf32": TF32}
VISUAL_WORKSPACE_BYTES = 4096   # casmvs_visual_panels

# name -> (restype, argtypes); must list every symbol include/casmvs.h declares
SIGNATURES = {
    "casmvs_version": (c_int, []),
    "casmvs_last_error": (c_char_p, []),
    "casmvs_device_check": (c_int, [c_int]),
    "casmvs_launch_count": (c_uint64, []),
    "casmvs_fallback_count": (c_uint64, []),
    "casmvs_conv3d_tensor_core": (c_int, [c_int] * 5),
    "casmvs_release_weight_images": (c_int, [c_void_p, c_size_t]),
    "casmvs_weight_cache_generation": (c_uint64, []),
    "casmvs_weight_image_count": (c_int, [c_void_p, c_size_t]),
    "casmvs_settle_weight_images": (c_int, []),
    "casmvs_warp_cost_workspace_bytes": (c_size_t, [c_int] * 6),
    "casmvs_warp_cost_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                     c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_void_p, c_size_t, c_void_p]),
    "casmvs_homo_warp_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                     c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "casmvs_packed_conv3d_weight_floats": (c_size_t, [c_int, c_int]),
    "casmvs_pack_conv3d_weights": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "casmvs_invalidate_weight_cache": (c_int, []),
    "casmvs_conv3d_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p,
                                  c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_int, c_int, c_int, c_void_p]),
    "casmvs_costreg_param_floats": (c_size_t, [c_int]),
    "casmvs_costreg_layer_info": (c_int, [c_int, c_int, POINTER(c_int), POINTER(c_int),
                                          POINTER(c_int), POINTER(c_int), POINTER(c_size_t),
                                          POINTER(c_size_t), POINTER(c_size_t)]),
    "casmvs_costreg_workspace_bytes": (c_size_t, [c_int] * 5),
    "casmvs_costreg_blocked_supported": (c_int, [c_int, c_int]),
    "casmvs_costreg_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                   c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "casmvs_costreg_tail_supported": (c_int, [c_int, c_int]),
    "casmvs_costreg_layer_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_int, c_int, c_int, c_void_p, c_size_t, c_int,
                                         c_void_p]),
    "casmvs_regress_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "casmvs_depth_hypotheses_fwd": (c_int, [c_void_p, c_int, c_float, c_float, c_void_p,
                                            c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "casmvs_uniform_hypotheses_fwd": (c_int, [c_float, c_float, c_void_p, c_void_p, c_void_p,
                                              c_int, c_int, c_int, c_int, c_void_p]),
    "casmvs_depth_first_fwd": (c_int, [c_void_p, c_int, c_float, c_float, c_void_p, c_void_p,
                                       c_int, c_int, c_int, c_int, c_void_p]),
    "casmvs_warp_cost_ladder_supported": (c_int, [c_int, c_int, c_int]),
    "casmvs_warp_cost_ladder_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p,
                                            c_float, c_void_p] + [c_int] * 8 + [c_void_p]),
    "casmvs_regress_ladder_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_float,
                                          c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "casmvs_inverse_hypotheses_fwd": (c_int, [c_void_p, c_float, c_void_p, c_float, c_void_p, c_float,
                                              c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "casmvs_regress_ladder_inverse_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p,
                                                  c_float, c_void_p, c_void_p, c_void_p] + [c_int] * 4
                                          + [c_void_p]),
    "casmvs_adaptive_hypotheses_fwd": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p]
                                       + [c_int] * 5 + [c_void_p]),
    "casmvs_regress_spread_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int] + [c_void_p] * 5
                                  + [c_int] * 4 + [c_void_p]),
    "casmvs_regress_ladder_spread_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_float]
                                         + [c_void_p] * 5 + [c_int] * 4 + [c_void_p]),
    "casmvs_warp_cost_ladder_step_fwd": (c_int, [c_void_p] * 5 + [c_int] * 8 + [c_void_p]),
    "casmvs_fpn_level_fwd":(c_int, [c_void_p] * 8 + [c_int] * 5 + [c_void_p]),
    "casmvs_fpn_merge_fwd": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_void_p]),
    "casmvs_conv2d_rgb8_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p] + [c_int] * 4 + [c_void_p]),
    "casmvs_conv2d_5x5s2_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p] + [c_int] * 6 + [c_void_p]),
    "casmvs_conv2d_5x5s2_fp32_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p] + [c_int] * 5 + [c_void_p]),
    "casmvs_bias_act_nhwc": (c_int, [c_void_p, c_void_p, c_float, c_size_t, c_int, c_int, c_void_p]),
    "casmvs_bias_lrelu_nhwc": (c_int, [c_void_p, c_void_p, c_float, c_size_t, c_int, c_void_p]),
    "casmvs_normalize_u8_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float),
                                        POINTER(c_float), c_void_p]),
    "casmvs_jitter_normalize_u8_fwd": (c_int, [c_void_p] * 4 + [c_int] * 3 + [POINTER(c_float),
                                                                            POINTER(c_float), c_void_p]),
    "casmvs_resize_u8_pil_fwd": (c_int, [c_void_p] * 3 + [c_int] * 5 + [c_void_p, c_void_p, c_int,
                                                                          c_void_p, c_void_p, c_int,
                                                                          c_void_p]),
    "casmvs_resize_u8_linear_fwd": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p] * 3),
    "casmvs_undistort_u8_fwd": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [POINTER(c_double),
                                                                         POINTER(c_double), c_void_p]),
    "casmvs_warp_cost_bwd": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_void_p]),
    "casmvs_conv3d_wgrad": (c_int, [c_void_p] * 3 + [c_int] * 10 + [c_void_p]),
    "casmvs_regress_bwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "casmvs_warp_cost_bwd_det_workspace_bytes": (c_size_t, [c_int] * 6),
    "casmvs_warp_cost_bwd_det": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_void_p, c_size_t, c_void_p]),
    "casmvs_conv3d_wgrad_det_workspace_bytes": (c_size_t, [c_int] * 6),
    "casmvs_conv3d_wgrad_det": (c_int, [c_void_p] * 3 + [c_int] * 10 + [c_void_p, c_size_t, c_void_p]),
    "casmvs_upsample2x_bilinear_bwd": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "casmvs_sl1_loss_workspace_bytes": (c_size_t, []),
    "casmvs_sl1_loss_fwd": (c_int, [POINTER(c_void_p)] * 3 + [POINTER(c_int), c_int, c_int]
                            + [c_void_p] * 4 + [c_size_t, c_void_p]),
    "casmvs_sl1_loss_bwd": (c_int, [POINTER(c_void_p)] * 3 + [POINTER(c_int), c_int, c_int]
                            + [c_void_p, c_void_p, POINTER(c_void_p), c_void_p]),
    "casmvs_photo_loss_workspace_bytes": (c_size_t, [c_int] * 4),
    "casmvs_photo_loss_fwd": (c_int, [c_void_p] * 3 + [POINTER(c_void_p), POINTER(c_float)]
                              + [c_int] * 6 + [c_float, POINTER(c_void_p)] + [c_void_p] * 3
                              + [POINTER(c_void_p)] * 3 + [c_void_p, c_size_t, c_void_p]),
    "casmvs_photo_loss_bwd": (c_int, [c_void_p] * 3 + [POINTER(c_void_p), POINTER(c_float)]
                              + [c_int] * 6 + [c_float, POINTER(c_void_p)]
                              + [c_void_p, c_void_p, POINTER(c_void_p), c_void_p]),
    "casmvs_geo_fuse_fwd":(c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    POINTER(c_float), POINTER(c_float), c_void_p, c_int, c_int,
                                    c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p]),
    "casmvs_geo_fuse_dynamic_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                            POINTER(c_float), POINTER(c_float), c_void_p, c_int,
                                            c_int, c_int, c_float, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "casmvs_pcd_cell_keys": (c_int, [c_void_p, c_int, c_double, c_double, c_double, c_double,
                                     c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "casmvs_pcd_thin_workspace_bytes": (c_size_t, [c_int, c_int]),
    "casmvs_pcd_thin_prepare": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                        c_void_p, c_size_t, c_void_p]),
    "casmvs_pcd_thin_round": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_double,
                                      c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "casmvs_pcd_capped_nn": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                     POINTER(c_double), c_double, POINTER(c_int), POINTER(c_double),
                                     POINTER(c_double), c_double, c_void_p, c_void_p]),
    "casmvs_pcd_capped_nn_index": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                           c_void_p, POINTER(c_double), c_double, POINTER(c_int),
                                           POINTER(c_double), POINTER(c_double), c_double,
                                           c_void_p, c_void_p, c_void_p, c_void_p]),
    "casmvs_pcd_knn_mean": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                    POINTER(c_double), c_double, POINTER(c_int), c_double,
                                    c_void_p, c_void_p, c_void_p]),
    "casmvs_pcd_sor_workspace_bytes": (c_size_t, [c_int]),
    "casmvs_pcd_sor_keep": (c_int, [c_void_p, c_int, c_double, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_size_t, c_void_p]),
    "casmvs_tnt_crop_blocks": (c_int, [c_int]),
    "casmvs_tnt_transform_crop": (c_int, [c_void_p, c_int, POINTER(c_double), c_int, c_double,
                                          c_double, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                          c_void_p]),
    "casmvs_tnt_compact": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                   c_void_p]),
    "casmvs_tnt_voxel_mean": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_tnt_icp_workspace_bytes": (c_size_t, [c_int]),
    "casmvs_tnt_icp_moments": (c_int, [c_void_p, c_int, c_void_p, c_void_p, POINTER(c_double),
                                       c_void_p, c_void_p, c_size_t, c_void_p]),
    "casmvs_view_scores_workspace_bytes": (c_size_t, [c_int, c_int, c_longlong]),
    "casmvs_view_scores_fwd": (c_int, [c_void_p] * 4 + [c_int, c_int, c_void_p, c_void_p, c_size_t,
                                                          c_void_p]),
    "casmvs_mesh_brick_keys": (c_int, [c_void_p, c_int, c_float, c_float, c_void_p, c_void_p,
                                       c_void_p]),
    "casmvs_mesh_brick_neighbors": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_mesh_integrate": (c_int, [c_void_p, c_int, c_float, c_float, c_void_p, c_void_p,
                                      POINTER(c_float), c_int, c_int, c_int, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    "casmvs_mesh_count": (c_int, [c_void_p, c_int] + [c_void_p] * 6),
    "casmvs_mesh_vertices": (c_int, [c_void_p, c_void_p, c_int, c_float] + [c_void_p] * 7),
    "casmvs_mesh_faces": (c_int, [c_void_p, c_int] + [c_void_p] * 6),
    "casmvs_poisson_workspace_bytes": (c_size_t, [c_longlong]),
    "casmvs_poisson_cell_keys": (c_int, [c_void_p, c_void_p, c_int, c_float] + [c_int] * 4
                                 + [c_void_p] * 3),
    "casmvs_poisson_cell_moments": (c_int, [c_void_p, c_void_p, c_int] + [c_double] * 3
                                    + [c_void_p] * 2),
    "casmvs_poisson_cell_normals": (c_int, [c_void_p] * 3 + [c_int] * 2 + [c_void_p] * 3),
    "casmvs_poisson_orient": (c_int, [c_void_p] * 3 + [c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_poisson_splat": (c_int, [c_void_p] * 5 + [c_int, c_float] + [c_int] * 3
                             + [c_void_p] * 4),
    "casmvs_poisson_rhs": (c_int, [c_void_p, c_int, c_float] + [c_void_p] * 4),
    "casmvs_poisson_residual": (c_int, [c_void_p, c_void_p, c_int, c_float] + [c_void_p] * 4),
    "casmvs_poisson_smooth": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_int,
                                      c_void_p]),
    "casmvs_poisson_mg_residual": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p,
                                           c_void_p]),
    "casmvs_poisson_restrict": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_poisson_prolong_add": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "casmvs_poisson_accumulate": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "casmvs_poisson_iso_sum": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float] + [c_int] * 3
                               + [c_void_p] * 3),
    "casmvs_poisson_trim": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "casmvs_poisson_brick_flags": (c_int, [c_void_p] + [c_int] * 10 + [c_void_p] * 2),
    "casmvs_poisson_fill_bricks": (c_int, [c_void_p, c_int] + [c_void_p] * 3 + [c_int] * 4
                                   + [c_void_p] * 3),
    "casmvs_poisson_fill_tsdf": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_double]
                                 + [c_int] * 4 + [c_void_p] * 2),
    "casmvs_poisson_screen_keys": (c_int, [c_void_p, c_int, c_float] + [c_int] * 4
                                   + [c_void_p] * 2),
    "casmvs_poisson_screen_moments": (c_int, [c_void_p] * 3 + [c_int, c_float] + [c_int] * 3
                                      + [c_void_p] * 2),
    "casmvs_poisson_screen_coarsen": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int,
                                              c_void_p, c_void_p]),
    "casmvs_poisson_screen_rhs": (c_int, [c_void_p] * 4 + [c_int, c_double] + [c_void_p] * 4),
    "casmvs_poisson_screen_stencil": (c_int, [c_void_p, c_int] + [c_void_p] * 3
                                      + [c_int, c_void_p, c_void_p, c_void_p]),
    "casmvs_poisson_screen_residual": (c_int, [c_void_p] * 5 + [c_int, c_float, c_double]
                                       + [c_void_p] * 4),
    "casmvs_poisson_screen_mg_residual": (c_int, [c_void_p] * 5 + [c_int, c_int, c_float, c_double]
                                          + [c_void_p] * 2),
    "casmvs_poisson_screen_smooth": (c_int, [c_void_p] * 5 + [c_int, c_int, c_float, c_double,
                                                              c_int, c_int, c_void_p]),
    "casmvs_simplify_clean": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_simplify_frozen": (c_int, [c_void_p, c_int] + [c_void_p] * 6),
    "casmvs_simplify_face_quadrics": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_simplify_vertex_quadrics": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 8),
    "casmvs_simplify_edge_costs": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 4
                                   + [c_int, c_void_p, c_int, c_double] + [c_void_p] * 7),
    "casmvs_simplify_select": (c_int, [c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_int]
                               + [c_void_p] * 6),
    "casmvs_simplify_collapse": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 6),
    "casmvs_simplify_remap_faces": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "casmvs_simplify_mark_used": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "casmvs_mesh_sample_count": (c_int, [c_void_p, c_void_p, c_int, c_double, c_void_p, c_void_p,
                                         c_void_p]),
    "casmvs_mesh_sample_points": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_longlong,
                                          c_void_p, c_void_p]),
    "casmvs_mesh_clean_face_area": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_mesh_clean_sums": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_mesh_clean_boundary": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int]
                                   + [c_void_p] * 5),
    "casmvs_mesh_clean_loop_sizes": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                             c_void_p]),
    "casmvs_mesh_clean_fill": (c_int, [c_void_p] * 5 + [c_int, c_int, c_void_p, c_void_p, c_int]
                               + [c_void_p] * 5),
    "casmvs_render_points_fwd":(c_int, [c_void_p, c_void_p, c_longlong, POINTER(c_float), c_int,
                                         c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "casmvs_render_mesh_workspace_bytes": (c_size_t, [c_int]),
    "casmvs_render_mesh_fwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, POINTER(c_float),
                                       POINTER(c_float), c_int, c_int, c_void_p, c_void_p, c_size_t,
                                       c_void_p, c_void_p, c_void_p]),
    "casmvs_render_mesh_keys": (c_int, [c_void_p, c_int, c_void_p, c_int, POINTER(c_float), c_int,
                                        c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "casmvs_render_textured_mesh_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                                c_void_p, c_int, c_int, POINTER(c_float), c_int,
                                                c_int, c_void_p, c_void_p, c_size_t, c_void_p,
                                                c_void_p, c_void_p]),
    "casmvs_texture_scores": (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(c_float),
                                      POINTER(c_double), POINTER(c_int), POINTER(c_int),
                                      POINTER(c_void_p), c_void_p, c_void_p, c_void_p]),
    "casmvs_texture_smooth": (c_int, [c_void_p] * 3 + [c_int, c_void_p, c_void_p, c_void_p]),
    "casmvs_texture_charts": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, POINTER(c_int),
                                      c_void_p]),
    "casmvs_texture_rects": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 5),
    "casmvs_texture_fill": (c_int, [c_void_p, c_int] + [c_void_p] * 4 + [c_int, c_void_p, c_void_p]),
    "casmvs_texture_uvs": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 4
                           + [c_int, c_void_p, c_void_p, c_void_p]),
    "casmvs_texture_level_keys": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "casmvs_texture_level_corners": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_texture_level_edges": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 6),
    "casmvs_texture_level_samples": (c_int, [c_void_p] * 6 + [c_int] + [c_void_p] * 5),
    "casmvs_texture_level_pairs": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_texture_level_system": (c_int, [c_void_p, c_void_p, c_longlong, c_int] + [c_void_p] * 7),
    "casmvs_texture_level_cg_workspace_bytes": (c_size_t, [c_int]),
    "casmvs_texture_level_cg": (c_int, [c_void_p] * 5 + [c_int, c_void_p, c_void_p, c_size_t, c_int,
                                                         c_double, c_int, POINTER(c_int),
                                                         POINTER(c_double), POINTER(c_int),
                                                         c_void_p]),
    "casmvs_texture_level_owners": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 4
                                    + [c_int, c_void_p, c_void_p]),
    "casmvs_texture_level_apply": (c_int, [c_void_p, c_longlong] + [c_void_p] * 6
                                   + [c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "casmvs_refine_grey": (c_int, [c_void_p, c_longlong, c_void_p, c_void_p]),
    "casmvs_refine_normals": (c_int, [c_void_p, c_int] + [c_void_p] * 5),
    "casmvs_refine_visibility": (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(c_float),
                                         POINTER(c_double), POINTER(c_int), POINTER(c_int),
                                         POINTER(c_void_p), c_void_p, c_int, c_void_p]),
    "casmvs_refine_select": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int]
                             + [c_void_p] * 6),
    "casmvs_refine_sweep": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 6
                            + [c_int] + [c_void_p] * 7),
    "casmvs_refine_smooth": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 5),
    "casmvs_refine_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "casmvs_visual_panels":(c_int, [c_void_p] * 5 + [c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "casmvs_nchw_to_nhwc":(c_int,[c_void_p, c_void_p, c_int, c_int, c_size_t, c_void_p]),
    "casmvs_nhwc_to_nchw": (c_int, [c_void_p, c_void_p, c_int, c_int, c_size_t, c_void_p]),
}

_lib = None


class CasMVSError(RuntimeError):
    pass


def load():
    """Load libcasmvs.so (once) and bind every symbol of the header."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise CasMVSError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (or `make -C casmvsnet_pl_b200/csrc`). There is no CPU/PyTorch "
            "fallback for the hot path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().casmvs_last_error()
        raise CasMVSError(f"{what}: {msg.decode() if msg else 'error'} (status {rc})")


def launch_count():
    return int(load().casmvs_launch_count())


def fallback_count():
    """tf32-mode layers that ran on the CUDA-core kernel because no wgmma kernel covers
    their shape (0 for the reference architecture)."""
    return int(load().casmvs_fallback_count())


def weight_cache_generation():
    return int(load().casmvs_weight_cache_generation())
