"""ctypes binding of libvtoonify_b200.so (the C-ABI declared in include/vtoonify_b200.h).

The product path fails loudly when the CUDA extension is missing: there is no CPU or PyTorch
fallback behind these calls.  The library is built in-tree by ``__graft_entry__.build()`` /
``vtoonify_b200/csrc/build.sh`` into ``vtoonify_b200/lib/``.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libvtoonify_b200.so")
ABI_VERSION = 7
VT_MAX_TAPS = 36
VT_ALIGN_MAX_RADIUS = 127   # include/vtoonify_b200.h: the longest Gaussian half-kernel of the alignment's blur
ACT_NONE, ACT_LRELU, ACT_RELU_TANH = 0, 1, 2


class VtError(RuntimeError):
    pass


class ConvDesc(Structure):
    _fields_ = [
        ("struct_size", c_int32), ("n_src", c_int32),
        ("src", c_void_p * 2), ("src_c", c_int32 * 2), ("src_cstride", c_int32 * 2),
        ("B", c_int32), ("H", c_int32), ("W", c_int32), ("Ho", c_int32), ("Wo", c_int32),
        ("stride", c_int32), ("taps", c_int32),
        ("tap_dy", c_int32 * VT_MAX_TAPS), ("tap_dx", c_int32 * VT_MAX_TAPS), ("tap_w", c_int32 * VT_MAX_TAPS),
        ("tap_phase", c_int32 * VT_MAX_TAPS), ("n_phase", c_int32), ("out_cpitch", c_int32), ("phase_off", c_int64 * 4),
        ("weight", c_void_p), ("wB", c_int32), ("w_taps", c_int32), ("w_cstride", c_int32), ("Cout", c_int32),
        ("out", c_void_p), ("out_sb", c_int64), ("out_sy", c_int64), ("out_sx", c_int64),
        ("bias", c_void_p), ("noise", c_void_p), ("noise_w", c_void_p),
        ("act", c_int32), ("slope", c_float), ("gain", c_float),
        ("res", c_void_p), ("alpha", c_float), ("beta", c_float),
        ("round_tf32", c_int32), ("reserved", c_int32),
        ("rgb_w", c_void_p), ("rgb_bias", c_void_p), ("rgb_skip", c_void_p), ("rgb_skip_kernel", c_void_p),
        ("rgb_out", c_void_p),
        ("slope_vec", c_void_p), ("weight_bf16x3", c_void_p), ("bf16x3_nstack", c_int32), ("reserved2", c_int32), ("src_scale", c_void_p * 2), ("src_affine", c_void_p * 2),
        ("split_fmt", c_int32), ("acc_scale", c_float),
        ("stats_ws", c_void_p), ("stats_ws_floats", c_int64),
    ]


class ConvWgradDesc(Structure):
    _fields_ = [
        ("struct_size", c_int32), ("B", c_int32), ("per_sample", c_int32), ("stride", c_int32),
        ("a", c_void_p), ("a_h", c_int32), ("a_w", c_int32), ("M", c_int32), ("a_cstride", c_int32),
        ("s", c_void_p), ("s_h", c_int32), ("s_w", c_int32), ("N", c_int32), ("s_cstride", c_int32),
        ("taps", c_int32), ("tap_dy", c_int32 * VT_MAX_TAPS), ("tap_dx", c_int32 * VT_MAX_TAPS),
        ("out", c_void_p), ("ws", c_void_p), ("ws_floats", c_int64),
    ]


class SmallNDesc(Structure):
    _fields_ = [
        ("struct_size", c_int32), ("n_planar", c_int32),
        ("planar", c_void_p), ("planar_weight", c_void_p),
        ("src", c_void_p), ("src_c", c_int32), ("src_cstride", c_int32),
        ("src2", c_void_p), ("src2_mode", c_int32),
        ("B", c_int32), ("H", c_int32), ("W", c_int32), ("taps", c_int32),
        ("tap_dy", c_int32 * VT_MAX_TAPS), ("tap_dx", c_int32 * VT_MAX_TAPS), ("tap_w", c_int32 * VT_MAX_TAPS),
        ("weight", c_void_p), ("wB", c_int32), ("w_taps", c_int32), ("w_cstride", c_int32), ("Cout", c_int32),
        ("bias", c_void_p), ("act", c_int32),
        ("skip", c_void_p), ("skip_kernel", c_void_p),
        ("out", c_void_p), ("mul_out", c_void_p), ("mul_src", c_void_p),
        ("mul_c", c_int32), ("round_tf32", c_int32),
        ("tap_const", c_void_p), ("src_mask", c_void_p), ("tsum", c_void_p), ("tsum_c", c_int32), ("reserved", c_int32),
    ]


# name -> (restype, argtypes); every symbol include/vtoonify_b200.h declares
_P = c_void_p
SYMBOLS = {
    "vt_abi_version": (c_int, []),
    "vt_last_error": (c_char_p, []),
    "vt_build_info": (c_char_p, []),
    "vt_launch_count": (c_int64, []),
    "vt_upfirdn2d_out_size": (c_int, [c_int] * 12 + [POINTER(c_int), POINTER(c_int)]),
    "vt_upfirdn2d_f32": (c_int, [_P, _P, _P, c_int64] + [c_int] * 12 + [_P]),
    "vt_fused_bias_act_f32": (c_int, [_P, _P, _P, c_int64, c_int64, c_int, c_float, c_float, _P]),
    "vt_fused_bias_act_grad_f32": (c_int, [_P, _P, _P, _P, c_int64, c_int64, c_int, c_float, c_float, _P]),
    "vt_channel_sum_ws_floats": (c_int64, [c_int]),
    "vt_channel_sum_f32": (c_int, [_P, _P, _P, c_int, c_int, c_int64, _P]),
    "vt_nchw_to_nhwc_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "vt_nhwc_to_nchw_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    "vt_linear_f32": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_float, c_float, c_int, _P]),
    "vt_pixelnorm_f32": (c_int, [_P, _P, c_int, c_int, _P]),
    "vt_modulate_weights_f32": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_int, _P]),
    "vt_fold_upconv_weights_f32": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_split_weights_bf16x3": (c_int, [_P, _P, c_int64, c_int, c_int, _P]),
    "vt_split_weights_f16x3": (c_int, [_P, _P, c_int64, c_int, c_float, _P]),
    "vt_conv2d_direct_f32": (c_int, [POINTER(ConvDesc), _P]),
    "vt_conv2d_tc_tf32": (c_int, [POINTER(ConvDesc), _P]),
    "vt_conv2d_tc_supported": (c_int, [POINTER(ConvDesc)]),
    "vt_conv2d_rs": (c_int, [POINTER(ConvDesc), c_float, _P]),
    "vt_conv2d_rs_supported": (c_int, [POINTER(ConvDesc)]),
    "vt_set_option": (c_int, [c_char_p, c_int]),
    "vt_conv2d_wgrad_ws_floats": (c_int64, [POINTER(ConvWgradDesc)]),
    "vt_conv2d_wgrad": (c_int, [POINTER(ConvWgradDesc), _P]),
    "vt_smalln_conv_f32": (c_int, [POINTER(SmallNDesc), _P]),
    "vt_affine_fold_weights_f32": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, _P]),
    "vt_fir_nhwc_f32": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, c_int,
                                c_float, c_float, c_int, _P]),
    "vt_instnorm_ws_bytes": (c_int64, [c_int, c_int64, c_int, c_int]),
    "vt_instnorm_finalize_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int64, c_float, _P]),
    "vt_instnorm_partials_floats": (c_int64, [c_int64, c_int, c_int]),
    "vt_conv2d_tc_stats_chunks": (c_int, [POINTER(ConvDesc)]),
    "vt_instnorm_stats_nhwc": (c_int, [_P, _P, c_int, c_int, c_int64, c_int, c_int, c_float, _P, _P, _P]),
    "vt_frame_s2d_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "vt_maxpool3x3s2_nhwc_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_maxpool2x2_nhwc_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_maxpool2x2_grad_nhwc_f32": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_lpips_head_ws_bytes": (c_int64, [c_int, c_int, POINTER(c_int64)]),
    "vt_lpips_head_nhwc": (c_int, [c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_int64), POINTER(c_int), c_int, _P, _P, _P]),
    "vt_lpips_head_grad_nhwc": (c_int, [_P, _P, _P, c_int, c_int64, c_int, _P, _P, _P]),
    "vt_augment_affine_plan": (c_int, [_P, c_int, c_int, c_int, POINTER(c_int)]),
    "vt_augment_affine_f32": (c_int, [_P, _P, _P, _P] + [c_int] * 11 + [_P]),
    "vt_raft_input_s2d_f32": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_raft_norm_relu_nhwc": (c_int, [_P, _P, _P, _P, _P, c_int, c_int64, c_int, _P]),
    "vt_raft_context_f32": (c_int, [_P, _P, _P, c_int64, c_int, c_int, _P]),
    "vt_raft_corr_pool_f32": (c_int, [_P, _P, c_int64, c_int, c_int, c_int64, _P]),
    "vt_raft_corr_lookup_f32": (c_int, [POINTER(c_void_p), POINTER(c_int64), c_int, c_int, _P, _P, c_int, c_int64, _P]),
    "vt_raft_fmap_pool_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_raft_corr_ondemand_f32": (c_int, [_P, c_int64, POINTER(c_void_p), c_int, c_int, c_int, _P, _P, c_int, _P]),
    "vt_raft_convf1_f32": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_raft_flow_f32": (c_int, [_P, _P, c_int, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_raft_gru_reset_f32": (c_int, [_P, _P, _P, c_int64, c_int, _P]),
    "vt_raft_gru_update_f32": (c_int, [_P, _P, _P, c_int64, c_int, _P]),
    "vt_raft_upsample_f32": (c_int, [_P, c_int, _P, _P, _P, c_int, c_int, c_int, _P]),
    "vt_flow_warp_f32": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_parsing_fuse_f32": (c_int, [POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_float), c_int, _P, c_int, c_int,
                                    c_int, _P]),
    "vt_parsing_fuse_down_f32": (c_int, [POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), POINTER(c_float), c_int, c_int, _P,
                                         c_int64, c_int, c_int, c_int, c_float, c_int, _P]),
    "vt_smooth_frame_prep_u8": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    "vt_resize_nearest_nhwc_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "vt_logits_readout_f32": (c_int, [_P, _P] + [c_int] * 10 + [c_float, c_int64, _P]),
    "vt_adain_affine_f32": (c_int, [_P, _P, _P, c_int, c_int, _P]),
    "vt_adain_apply_nhwc": (c_int, [_P, _P, c_int, c_int, c_int64, c_int, c_int, _P, _P, _P, c_int, _P]),
    "vt_act_grad_ws_bytes": (c_int64, [c_int, c_int64, c_int]),
    "vt_adain_grad_stats_nhwc": (c_int, [_P, _P, _P, c_int, c_int64, c_int, _P, _P, _P]),
    "vt_act_grad_nhwc": (c_int, [_P, _P, c_float, c_float, _P, c_float, _P, _P, _P, _P, c_int, c_int64, c_int, _P, _P, _P, _P]),
    "vt_torgb_gate_grad_nhwc": (c_int, [_P, _P, _P, c_int, c_int, _P, c_float, c_float, c_int, c_int64, c_int, _P, _P]),
    "vt_fusion_mask_grad_ws_bytes": (c_int64, [c_int, c_int64]),
    "vt_fusion_mask_grad_nhwc": (c_int, [_P, _P, _P, _P, c_int, c_int64, c_int, _P, _P, _P, _P]),
    "vt_fusion_adain_grad_stats_nhwc": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, _P]),
    "vt_fusion_input_grad_nhwc": (c_int, [_P] * 10 + [c_int, c_int, c_int, c_int, _P, _P, _P]),
    "vt_mbstd_nhwc_f32": (c_int, [_P, _P, c_int, c_int, c_int64, c_int, c_int, _P]),
    "vt_mbstd_grad_nhwc_f32": (c_int, [_P, _P, _P, c_int, c_int, c_int64, c_int, c_int, _P]),
    "vt_gate_shortcut_add_nhwc": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "vt_bilinear_add_nhwc": (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    "vt_axpby_f32": (c_int, [_P, _P, _P, c_int64, c_float, c_float, c_int, _P]),
    "vt_frame_blur4_u8": (c_int, [_P, _P, c_int, c_int, c_int, _P]),
    "vt_frame_resize_crop_u8": (c_int, [_P, _P] + [c_int] * 9 + [_P, _P, _P]),
    "vt_align_lanczos_u8": (c_int, [_P, c_int64, c_int, c_int, _P, c_int, c_int, _P, c_int, _P]),
    "vt_align_blur_rows_f32": (c_int, [_P, c_int64, c_int, c_int, _P, _P, _P, c_int, _P]),
    "vt_align_blur_cols_f32": (c_int, [_P, _P, c_int, c_int, _P, c_int, _P, c_int64, c_int, c_int, _P, _P]),
    "vt_align_median_ws_bytes": (c_int64, []),
    "vt_align_median_f32": (c_int, [_P, c_int64, _P, _P, _P]),
    "vt_align_finish_u8": (c_int, [_P, _P, _P, c_int, c_int, _P, _P]),
    "vt_align_warp_u8": (c_int, [_P, c_int64, c_int, c_int, _P, _P, c_int, _P]),
    "vt_frame_u8_to_f32": (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int64, _P]),
    "vt_f32_to_frame_u8": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
}

_lib = None


def load():
    """Load the shared library (once) and bind every declared symbol. Raises VtError if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VtError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or vtoonify_b200/csrc/build.sh). vtoonify_b200 has no CPU / PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.vt_abi_version() != ABI_VERSION:
        raise VtError(f"ABI mismatch: library reports {lib.vt_abi_version()}, binding expects {ABI_VERSION}")
    for env, key in (("VT_TC_MODE", b"tc_mode"), ("VT_TC_MT", b"tc_mt"), ("VT_TC_TGROUP", b"tc_tgroup"),
                     ("VT_TC_STAGE_POLICY", b"tc_stage_policy"), ("VT_TC_HALO_PCT", b"tc_halo_pct"), ("VT_TC_M_MAJOR", b"tc_m_major"),
                     ("VT_INSTNORM_CHUNKS", b"instnorm_chunks")):
        if os.environ.get(env) is not None and os.environ.get(env) != "":
            lib.vt_set_option(key, int(os.environ[env]))      # tuning experiments only
    _lib = lib
    return lib


def check(status):
    if status != 0:
        raise VtError(load().vt_last_error().decode("utf-8", "replace"))


def launch_count():
    return int(load().vt_launch_count())
