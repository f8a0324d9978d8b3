"""ctypes binding of libsemseg_b200.so (the C-ABI declared in include/semseg_b200.h).

The product path has no CPU fallback: if the library is missing or an entry point fails, this module
raises. Nothing under oracle/ is ever imported from here.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libsemseg_b200.so")

MAX_TAPS = 9
EPI_RAW, EPI_AFFINE, EPI_F32 = 0, 1, 2
PSA_DENSE, PSA_NO_SOFTMAX = 1, 2          # form bits of semseg_psa_attend_ex / semseg_psa_attend_bwd_attn_ex

c_int = ctypes.c_int
c_i32 = ctypes.c_int32
c_vp = ctypes.c_void_p
c_f = ctypes.c_float
c_ll = ctypes.c_longlong
I9 = c_i32 * MAX_TAPS


class PackItem(ctypes.Structure):
    """struct semseg_pack_item (include/semseg_b200.h)."""
    _fields_ = [
        ("w", c_vp), ("wf", c_vp), ("wd", c_vp), ("wp", c_vp),
        ("Cout", c_i32), ("Cin", c_i32), ("taps", c_i32),
        ("cols_f", c_i32), ("cols_d", c_i32),
        ("tile0", c_i32), ("tiles_ci", c_i32),
        ("split", c_i32),
    ]


class SgdItem(ctypes.Structure):
    """struct semseg_sgd_item (include/semseg_b200.h)."""
    _fields_ = [("w", c_vp), ("buf", c_vp), ("n", c_ll), ("group", c_i32), ("chunk0", c_i32), ("first", c_i32),
                ("reserved", c_i32)]


EMA_LERP_F32, EMA_COPY_I64 = 0, 1        # semseg_ema_item.kind


class EmaItem(ctypes.Structure):
    """struct semseg_ema_item (include/semseg_b200.h)."""
    _fields_ = [("shadow", c_vp), ("source", c_vp), ("n", c_ll), ("kind", c_i32), ("chunk0", c_i32)]


class SgdHyper(ctypes.Structure):
    """struct semseg_sgd_hyper (include/semseg_b200.h)."""
    _fields_ = [("lr", c_f * 16), ("momentum", c_f * 16), ("weight_decay", c_f * 16), ("dampening", c_f * 16),
                ("nesterov", c_i32)]


class ConvDesc(ctypes.Structure):
    """struct semseg_conv_desc (include/semseg_b200.h)."""
    _fields_ = [
        ("N", c_i32), ("H", c_i32), ("W", c_i32),
        ("Cin", c_i32), ("Cout", c_i32),
        ("x", c_vp),
        ("Nin", c_i32), ("Hin", c_i32), ("Win", c_i32), ("x_pitch", c_i32),
        ("w", c_vp),
        ("n_wtaps", c_i32), ("w_rows", c_i32), ("w_cols", c_i32),
        ("taps", c_i32),
        ("dh", I9), ("dw", I9), ("wtap", I9),
        ("img_mul", c_i32), ("img_add", I9),
        ("epi_mode", c_i32), ("relu", c_i32),
        ("y", c_vp), ("y_pitch", c_i32),
        ("scale", c_vp), ("shift", c_vp),
        ("residual", c_vp), ("res_pitch", c_i32),
        ("out_f32", c_vp), ("out_pitch", c_i32),
        ("stats_partial", c_vp),
        ("x_lo", c_vp), ("y_lo", c_vp), ("residual_lo", c_vp),
        ("w_split", c_i32),
        ("k_slices", c_i32), ("slice_stride", ctypes.c_int64),
    ]


class WgradDesc(ctypes.Structure):
    """struct semseg_wgrad_desc (include/semseg_b200.h)."""
    _fields_ = [
        ("N", c_i32), ("H", c_i32), ("W", c_i32),
        ("Cin", c_i32), ("Cout", c_i32),
        ("x", c_vp),
        ("Nin", c_i32), ("Hin", c_i32), ("Win", c_i32), ("x_pitch", c_i32),
        ("dy", c_vp), ("dy_pitch", c_i32),
        ("taps", c_i32),
        ("dh", I9), ("dw", I9),
        ("img_mul", c_i32), ("img_add", I9),
        ("dw_partial", c_vp),
        ("n_splits", c_i32),
        ("x_lo", c_vp), ("dy_lo", c_vp),
    ]


class AugmentDesc(ctypes.Structure):
    """struct semseg_augment_desc (include/semseg_b200.h): one sample of semseg_augment."""
    _fields_ = [("img_off", c_ll), ("lab_off", c_ll), ("h", c_i32), ("w", c_i32), ("rh", c_i32), ("rw", c_i32),
                ("scale_y", ctypes.c_double), ("scale_x", ctypes.c_double), ("m", ctypes.c_double * 6),
                ("rotate", c_i32), ("blur", c_i32), ("flip", c_i32), ("pad_top", c_i32), ("pad_left", c_i32),
                ("off_y", c_i32), ("off_x", c_i32), ("reserved", c_i32)]


# name -> (restype, argtypes); must list every symbol include/semseg_b200.h declares
# (tests/test_abi.py parses the header and checks both directions).
SIGNATURES = {
    "semseg_last_error": (ctypes.c_char_p, []),
    "semseg_abi_version": (c_int, []),
    "semseg_launch_count": (c_ll, []),
    "semseg_psamask_fwd": (c_int, [c_int, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_psamask_bwd": (c_int, [c_int, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_psa_attend": (c_int, [c_int, c_int, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int,
                                  c_int, c_int, c_int, c_int, c_f, c_vp]),
    "semseg_psa_attend_bwd_attn": (c_int, [c_int, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp,
                                           c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_f, c_vp]),
    "semseg_psa_attend_ex": (c_int, [c_int, c_int, c_int, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int,
                                     c_int, c_int, c_int, c_int, c_int, c_int, c_f, c_vp]),
    "semseg_psa_attend_bwd_attn_ex": (c_int, [c_int, c_int, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_int,
                                              c_vp, c_vp, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_f,
                                              c_vp]),
    "semseg_conv_stats_rows": (c_int, [c_int, c_int, c_int, c_int]),
    "semseg_conv_k_slices": (c_int, [c_int, c_int, c_int]),
    "semseg_conv_splitk_rows": (c_int, [c_int]),
    "semseg_conv_splitk_finish": (c_int, [c_vp, c_int, c_ll, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp,
                                          c_int, c_vp, c_vp, c_int, c_vp, c_vp]),
    "semseg_conv_fprop": (c_int, [ctypes.POINTER(ConvDesc), c_vp]),
    "semseg_conv_wgrad_splits": (c_int, [ctypes.POINTER(WgradDesc)]),
    "semseg_conv_wgrad": (c_int, [ctypes.POINTER(WgradDesc), c_vp]),
    "semseg_wgrad_reduce": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_vp]),
    "semseg_pack_weights_multi": (c_int, [c_vp, c_int, c_int, c_int, c_vp]),
    "semseg_sgd_chunk_elems": (c_int, []),
    "semseg_sgd_multi": (c_int, [c_vp, c_vp, c_int, c_int, ctypes.POINTER(SgdHyper), c_vp]),
    "semseg_ema_multi": (c_int, [c_vp, c_int, c_int, ctypes.c_double, c_vp]),
    "semseg_iou_hist": (c_int, [c_vp, c_vp, ctypes.c_longlong, c_int, ctypes.c_longlong, c_int, c_vp, c_vp]),
    "semseg_im2col3x3s2": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "semseg_stem_dgrad3x3s2": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_int,
                                       c_vp, c_vp]),
    "semseg_nchw_f32_to_nhwc_bf16": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_nhwc_bf16_to_nchw_f32": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_nhwc_f32_to_nchw_f32": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_space_to_phases": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "semseg_phases_to_space": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "semseg_bn_merge_partials": (c_int, [c_vp, c_int, c_int, c_vp, c_vp]),
    "semseg_bn_workspace_floats": (c_ll, [c_int, c_int]),
    "semseg_bn_finalize": (c_int, [c_vp, c_int, c_int, c_vp, c_vp, c_f, c_f, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_bn_finalize_partials": (c_int, [c_vp, c_int, c_int, c_vp, c_vp, c_f, c_f, c_vp, c_vp, c_vp, c_vp,
                                            c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "semseg_bn_fold_eval": (c_int, [c_vp, c_vp, c_vp, c_vp, c_f, c_int, c_vp, c_vp]),
    "semseg_bn_apply": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                c_vp]),
    "semseg_bn_bwd_reduce": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_int,
                                     c_int, c_vp, c_ll, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "semseg_bn_bwd_apply": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
                                    c_f, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp]),
    "semseg_bn_bwd_frozen": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
                                     c_f, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_ll, c_vp,
                                     c_vp]),
    "semseg_add_act": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_int, c_int, c_int, c_vp]),
    "semseg_scale_nc": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_fp_fork": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_fp_fold": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_fp_fork_prefix": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_fp_fold_prefix": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_f32_to_act": (c_int, [c_vp, c_int, c_vp, c_vp, c_int, c_ll, c_int, c_int, c_vp]),
    "semseg_act_to_f32": (c_int, [c_vp, c_vp, c_int, c_vp, c_int, c_ll, c_int, c_vp]),
    "semseg_maxpool3x3s2_fwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_maxpool3x3s2_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp]),
    "semseg_ppm_pool": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_vp]),
    "semseg_ppm_pool_bwd": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp, c_vp,
                                    c_int, c_vp]),
    "semseg_ppm_upsample_concat": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                           c_int, c_vp, c_vp, c_int, c_vp]),
    "semseg_ppm_upsample_bwd": (c_int, [c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                        c_vp]),
    "semseg_resize_bilinear_fwd": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int,
                                           c_vp]),
    "semseg_resize_bilinear_bwd": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_int,
                                           c_vp]),
    "semseg_upsample_ce_workspace_floats": (c_ll, [c_int, c_int, c_int]),
    "semseg_upsample_ce_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_vp,
                                       c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_vp,
                                       c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_zoom_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_zoom_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                            c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_zoom_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_zoom_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                            c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_ohem_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_ohem_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                            c_f, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_ohem_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_ohem_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                            c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_weighted_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_weighted_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                                c_int, c_vp, c_f, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_weighted_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_weighted_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                                c_int, c_vp, c_f, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_ohem_weighted_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int,
                                                     c_int, c_int, c_f, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                     c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_ohem_weighted_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int,
                                                     c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                     c_vp]),
    "semseg_upsample_ce_dice_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_dice_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                            c_f, c_f, c_f, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_dice_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_dice_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                            c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_rmi_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_rmi_table_floats": (c_ll, [c_int, c_int]),
    "semseg_upsample_ce_rmi_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                           c_f, c_f, c_f, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_rmi_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_rmi_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                           c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_focal_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_focal_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                             c_vp, c_f, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_focal_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_focal_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_int,
                                             c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_lovasz_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_lovasz_fwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                              c_int, c_int, c_int, c_f, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_ce_lovasz_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_ce_lovasz_bwd": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                              c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_kd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int]),
    "semseg_upsample_kd_fwd": (c_int, [c_vp, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_f,
                                       c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_kd_bwd_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int, c_int]),
    "semseg_upsample_kd_bwd": (c_int, [c_vp, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_f,
                                       c_f, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_pl_workspace_floats": (c_ll, [c_int, c_int, c_int, c_int]),
    "semseg_upsample_pl_fwd": (c_int, [c_vp, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int,
                                       c_int, c_f, c_f, c_f, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_upsample_pl_mix_fwd": (c_int, [c_vp, c_int, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int,
                                           c_int, c_int, c_f, c_f, c_f, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                           c_vp]),
    "semseg_mix_argmax_x8": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "semseg_mix_select": (c_int, [c_vp, c_int, c_vp, c_int, c_int, c_vp, c_vp]),
    "semseg_mix_apply": (c_int, [c_int, c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_vp, c_int,
                                 ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                 c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_strong_augment": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_vp, c_int] + [ctypes.c_double] * 9 +
                              [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "semseg_segsort_u32_pairs_workspace_bytes": (c_ll, [c_int, c_ll]),
    "semseg_segsort_u32_pairs": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_ll, c_vp, c_vp, c_vp]),
    "semseg_window_scores": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_vp]),
    "semseg_window_accumulate": (c_int, [c_vp, c_int, c_int, c_int, c_vp, c_int, c_vp, c_int, c_int, c_int, c_int,
                                         c_int, c_int, c_int, c_vp, c_vp]),
    "semseg_window_resize_add": (c_int, [c_vp, c_int, c_int, c_int, c_vp, c_int, c_int, c_vp]),
    "semseg_augment": (c_int, [c_vp, c_ll, ctypes.POINTER(AugmentDesc), c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int,
                               c_vp, c_vp, c_vp]),
}

_lib = None


class SemsegError(RuntimeError):
    pass


def load():
    """Load the shared library (once) and attach signatures. Raises if it is missing: no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SemsegError(
            "libsemseg_b200.so is not built (%s). Run `python -m semseg_b200.build` "
            "(or __graft_entry__.build()); there is no CPU/PyTorch fallback for this path." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here means header/library drift: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status, what):
    if status != 0:
        msg = load().semseg_last_error()
        raise SemsegError("%s failed (%d): %s" % (what, status, msg.decode() if msg else "?"))


def launch_count():
    return int(load().semseg_launch_count())
