"""ctypes binding of libmqdet_b200.so (the C-ABI boundary, see include/mqdet_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` (``make -C mqdet_b200/csrc``).  There is no
CPU or PyTorch fallback: if the shared object is missing, loading raises.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmqdet_b200.so")

F16, F32 = 0, 1
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2
VEC_NONE, VEC_SCALAR, VEC_PER_COL, VEC_PER_ROW = 0, 1, 2, 3
IMPL_TC, IMPL_SIMT, IMPL_TC_ONESHOT = 0, 1, 2


class GemmArgs(ctypes.Structure):
    """Mirror of ``mqdet_gemm_args`` (include/mqdet_b200.h)."""

    _fields_ = [
        ("A", c_void_p), ("B", c_void_p),
        ("M", c_int64), ("N", c_int64), ("K", c_int64),
        ("lda", c_int64), ("ldb", c_int64),
        ("nb1", c_int64), ("nb2", c_int64),
        ("a_b1", c_int64), ("a_b2", c_int64), ("b_b1", c_int64), ("b_b2", c_int64),
        ("C", c_void_p), ("c_dtype", c_int32),
        ("ldc", c_int64), ("c_b1", c_int64), ("c_b2", c_int64),
        ("alpha", c_float), ("scale_after_bias", c_int32),
        ("bias", c_void_p), ("bias_mode", c_int32), ("bias_b1", c_int64), ("bias_b2", c_int64),
        ("act", c_int32), ("clamp", c_float),
        ("gate", c_void_p), ("gate_mode", c_int32), ("gate_tanh", c_int32),
        ("R", c_void_p), ("r_dtype", c_int32), ("ldr", c_int64), ("r_b1", c_int64), ("r_b2", c_int64),
    ]


# name -> (restype, argtypes); every symbol include/mqdet_b200.h declares must appear here
# (tests/test_abi.py checks the two lists against each other).
SIGNATURES = {
    "mqdet_last_error": (c_char_p, []),
    "mqdet_version": (c_int, []),
    "mqdet_reserve_sms": (c_int, [c_int]),
    "mqdet_gemm_f16": (c_int, [POINTER(GemmArgs), c_int, c_void_p]),
    "mqdet_layernorm": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p, c_float, c_int64, c_int64, c_void_p,
                                c_void_p, c_int64, c_int64, c_void_p]),
    "mqdet_swin_mlp_f16": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_void_p]),
    "mqdet_add_layernorm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int64, c_int64, c_void_p,
                                    c_void_p, c_float, c_void_p]),
    "mqdet_gcp_sparse_attn": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64,
                                      c_int64, c_int64, c_void_p]),
    "mqdet_gcp_gate_residual_ln": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_float, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mqdet_gcp_build_index": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_softmax_rows": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64, c_float,
                                   c_void_p, c_int64, c_float, c_float, c_void_p]),
    "mqdet_biattn_text_vn": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64,
                                     c_int64, c_int64, c_void_p, c_void_p, c_int64, c_float, c_void_p, c_int64, c_int64, c_int64,
                                     c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "mqdet_biattn_image_workspace_floats": (c_int64, [c_int64, c_int64, c_int64, c_int64]),
    "mqdet_biattn_image": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_void_p,
                                   c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_float,
                                   c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "mqdet_l2norm_rowdot": (c_int, [c_void_p, c_int64, c_int64, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    "mqdet_cast_f32_f16": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "mqdet_cast_f16_f32": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "mqdet_contrastive_mask": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "mqdet_argsort_desc": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "mqdet_ml_nms_workspace_bytes": (c_int64, [c_int64]),
    "mqdet_global_max_workspace_floats": (c_int64, [c_int64]),
    "mqdet_global_max_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_sum_splits_cast": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "mqdet_softmax_rows_shifted_supported": (c_int, [c_int64, c_int64]),
    "mqdet_softmax_rows_shifted": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_int64, c_float,
                                           c_float, c_void_p, c_int64, c_float, c_float, c_void_p]),
    "mqdet_shift_clamp_f32": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_float, c_float, c_void_p]),
    "mqdet_row_max_f32": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_topk_desc": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_gather_rows_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p, c_void_p]),
    "mqdet_dcn_conv": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_void_p]),
    "mqdet_dcn_cols": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int, c_void_p,
                               c_void_p]),
    "mqdet_conv3x3_small": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p,
                                    c_int64, c_void_p]),
    "mqdet_chan_stats_floats": (c_int64, [c_int64, c_int64, c_int64]),
    "mqdet_chan_stats": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_gn_attn": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p, c_void_p, c_float,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mqdet_dyconv_combine_chunks": (c_int64, []),
    "mqdet_dyconv_combine": (c_int, [c_void_p] * 9 + [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_dyrelu_coef": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_void_p]),
    "mqdet_dyrelu_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_atss_workspace_bytes": (c_int64, [c_void_p, c_int64, c_int64, c_int64]),
    "mqdet_atss_candidates": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64,
                                      c_void_p, c_int64,
                                      c_void_p, c_void_p, c_void_p, c_int64, c_float, c_int64, c_int64, c_float, c_float,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "mqdet_ml_nms_batched_workspace_bytes": (c_int64, [c_int64, c_int64]),
    "mqdet_ml_nms_batched": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_float, c_int64, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    "mqdet_gather_detections": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64,
                                        c_int64, c_void_p, c_void_p]),
    "mqdet_roi_align_levels": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64,
                                       c_int, c_void_p, c_void_p, c_void_p]),
    "mqdet_roi_align_levels_counted": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_int64,
                                               c_int64, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "mqdet_ms_deform_attn": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64,
                                     c_int64, c_int64, c_int64, c_void_p, c_int, c_void_p]),
    "mqdet_dense_cross_attn": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64,
                                       c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p]),
    "mqdet_anchors": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_float, c_void_p, c_float, c_float, c_void_p]),
    "mqdet_patchify4": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_swin_window_attn": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64,
                                       c_float, c_void_p, c_void_p]),
    "mqdet_patch_merge_ln": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_float, c_void_p,
                                     c_void_p]),
    "mqdet_upsample_add": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p,
                                   c_void_p]),
    "mqdet_im2col3x3": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p, c_void_p]),
    "mqdet_avgpool2_levels": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_ml_nms": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_int64, c_void_p, c_void_p,
                             c_void_p, c_void_p]),
    "mqdet_add_cast": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_groupnorm_rows_workspace_floats": (c_int64, [c_int64, c_int64]),
    "mqdet_groupnorm_rows": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_float, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    "mqdet_box_refine_sine": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    "mqdet_gdino_detections_workspace_floats": (c_int64, [c_int64, c_int64]),
    "mqdet_gdino_detections": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_void_p,
                                       c_float, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_transpose_cast": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int64, c_float, c_void_p, c_int64, c_void_p]),
    "mqdet_layernorm_bwd_workspace_floats": (c_int64, [c_int64, c_int64]),
    "mqdet_layernorm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int64, c_int64, c_void_p, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    "mqdet_transpose_cast_batched": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_float,
                                             c_void_p, c_int64, c_void_p]),
    "mqdet_softmax_bwd_rows": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p, c_int64,
                                       c_void_p]),
    "mqdet_gelu_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "mqdet_gcp_gate_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                                   c_void_p]),
    "mqdet_colsum_weighted_workspace_floats": (c_int64, [c_int64]),
    "mqdet_colsum_weighted": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_gcp_sparse_attn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64,
                                          c_void_p, c_void_p, c_void_p]),
    "mqdet_reduce_workspace_floats": (c_int64, []),
    "mqdet_dot_sum": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_float, c_void_p, c_void_p, c_void_p]),
    "mqdet_scale_cast": (c_int, [c_void_p, c_void_p, c_int, c_float, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_token_focal_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_int64, c_int64, c_int64, c_float, c_void_p,
                                       c_void_p, c_void_p, c_void_p]),
    "mqdet_sqnorm_partials": (c_int, [c_void_p, c_int64, c_void_p, c_int64, POINTER(c_int64), c_void_p]),
    "mqdet_clip_coef": (c_int, [c_void_p, c_int64, c_float, c_void_p, c_void_p]),
    "mqdet_adamw_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float, c_float, c_float, c_int64,
                                 c_void_p, c_void_p]),
    "mqdet_atss_assign_workspace_bytes": (c_int64, [c_int64, c_int64]),
    "mqdet_atss_assign": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_void_p]),
    "mqdet_atss_loss_workspace_floats": (c_int64, [c_int64, c_int64]),
    "mqdet_atss_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                                c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_float, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_void_p]),
    "mqdet_gdino_match_cost": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64,
                                       c_float, c_float, c_float, c_float, c_void_p, c_void_p, c_void_p]),
    "mqdet_linear_sum_assignment_workspace_bytes": (c_int64, [c_int64, c_int64, c_int64]),
    "mqdet_linear_sum_assignment": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_gdino_set_loss_workspace_floats": (c_int64, [c_int64, c_int64, c_int64]),
    "mqdet_gdino_set_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64,
                                     c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_float, c_float, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    "mqdet_hflip_pad": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_bbox_aug_collect": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_float, c_int, c_float,
                                       c_float, c_float, c_float, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                                       c_void_p]),
    "mqdet_bbox_aug_collect_packed": (c_int, [c_void_p, c_int64, c_int64, c_int, c_float, c_int, c_float, c_float, c_float, c_float,
                                              c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_nms_by_class_workspace_bytes": (c_int64, [c_int64, c_int64, c_int64]),
    "mqdet_nms_by_class": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_float,
                                   c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "mqdet_resize_coeffs_ksize": (c_int64, [c_int64, c_int64]),
    "mqdet_resize_coeffs": (c_int, [c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_test_transform": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_int,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mqdet_mask_prompt_tokens": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_query_candidates": (c_int, [c_void_p, c_int64, c_int64, c_float, c_float, c_int64, c_int64, c_void_p, c_void_p, c_int64,
                                       c_void_p, c_void_p, c_void_p]),
    "mqdet_query_bank_norms": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p]),
    "mqdet_query_bank_update": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64,
                                        c_float, c_void_p]),
    "mqdet_lvis_collect":(c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int,
                                   c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p,
                                   c_void_p]),
    "mqdet_lvis_cut_workspace_bytes": (c_int64, [c_int64, c_int64]),
    "mqdet_lvis_cut": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int64, c_int64, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mqdet_lvis_evaluate_workspace_bytes": (c_int64, [c_int64, c_int64]),
    "mqdet_lvis_evaluate": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p, c_int64,
                                    c_void_p, c_int64, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
}

_lib = None


class MqdetError(RuntimeError):
    """Raised when a C-ABI call returns a negative code (mirrors the reference's AT_ERROR -> RuntimeError)."""


# tools/breakdown.py sets this to a list: every C-ABI call is then bracketed by CUDA events -> (symbol, e0, e1)
CALL_PROFILE = None


class _Profiled:
    """Proxy over the CDLL that times each entry point on the current stream (diagnostics only)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name not in SIGNATURES or SIGNATURES[name][0] is not c_int or not SIGNATURES[name][1]:
            return fn

        def timed(*a):
            import torch
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*a)
            e1.record()
            CALL_PROFILE.append((name, e0, e1))
            return rc
        return timed


def load():
    """Load the shared library and bind every declared symbol (raises if the build is missing)."""
    global _lib
    if _lib is not None:
        return _Profiled(_lib) if CALL_PROFILE is not None else _lib
    if not os.path.exists(LIB_PATH):
        raise MqdetError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the mqdet_b200 hot path)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().mqdet_last_error()
        raise MqdetError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")
