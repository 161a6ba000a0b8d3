"""ctypes binding of libctrlora_b200.so (the C ABI declared in include/ctrlora_b200.h).

There is no CPU fallback: if the library is missing or a call fails, this module raises.
"""
import ctypes as C
import os

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libctrlora_b200.so")
_lib = None

c_void_p, c_int, c_ll, c_float = C.c_void_p, C.c_int, C.c_longlong, C.c_float


class GemmArgs(C.Structure):
    """Mirror of `struct ctrlora_gemm_args`."""
    _fields_ = [
        ("a", c_void_p), ("a_b", c_int), ("a_h", c_int), ("a_w", c_int), ("a_c", c_int), ("a_ld", c_ll),
        ("w", c_void_p), ("kh", c_int), ("kw", c_int), ("pad", c_int),
        ("a2", c_void_p), ("a2_c", c_int), ("a2_ld", c_ll), ("w2", c_void_p),
        ("n", c_int), ("block_n", c_int), ("geglu", c_int),
        ("out", c_void_p * 3), ("seg_width", c_int), ("transposed", c_int * 3),
        ("ldc", c_int), ("out_f32", c_int),
        ("bias", c_void_p), ("rowbias", c_void_p), ("rows_per_img", c_int), ("rowbias_ld", c_int),
        ("residual", c_void_p), ("ldr", c_int), ("residual_f32", c_int), ("out_scale", c_float),
        ("head_dim", c_int), ("tok_pad", c_int), ("bf16", c_int),
        ("split_k", c_int), ("splitk_ws", c_void_p), ("splitk_ws_bytes", c_ll),
        ("splitk_counters", c_void_p), ("splitk_counters_len", c_int),
        ("dup_out", c_void_p), ("dup_ld", c_int), ("force_single_cta", c_int),
        ("group_b", c_int), ("w_hi", c_void_p), ("bias_hi", c_void_p), ("rowbias_hi", c_void_p), ("w2_hi", c_void_p),
        ("relu", c_int),
    ]


class GroupNormArgs(C.Structure):
    """Mirror of `struct ctrlora_groupnorm_args`."""
    _fields_ = [
        ("x1", c_void_p), ("add1", c_void_p), ("add1_scale", c_float), ("c1", c_int), ("ld1", c_ll),
        ("x2", c_void_p), ("add2", c_void_p), ("add2_scale", c_float), ("c2", c_int), ("ld2", c_ll),
        ("batch", c_int), ("hw", c_int), ("groups", c_int),
        ("gamma", c_void_p), ("beta", c_void_p), ("eps", c_float), ("silu", c_int),
        ("y", c_void_p), ("raw_out", c_void_p), ("stats_ws", c_void_p),
        ("partial_ws", c_void_p), ("partial_ws_floats", c_ll), ("partial_counters", c_void_p), ("partial_counters_len", c_int),
        ("gamma_hi", c_void_p), ("beta_hi", c_void_p), ("group_b", c_int),
    ]


class CtrloraError(RuntimeError):
    pass


_STATUS = {1: "bad argument", 2: "CUDA error", 3: "tensor-map encode error", 4: "unsupported"}
STATUS_UNSUPPORTED = 4


def lib_path():
    return _LIB_PATH


def load():
    """Load the shared library (building is the job of ctrlora_b200.build / __graft_entry__.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise CtrloraError(
                f"{_LIB_PATH} is missing: run `python -m ctrlora_b200.build` (needs nvcc). "
                "ctrlora_b200 has no CPU or PyTorch fallback.")
        _lib = C.CDLL(_LIB_PATH)
        _declare(_lib)
    return _lib


_P, _I, _L, _F = c_void_p, c_int, c_ll, c_float
_D = C.c_double
_ARGTYPES = {
    "ctrlora_gemm_f16": [_P, _P],
    "ctrlora_gemm_f16_simt": [_P, _P],
    "ctrlora_groupnorm_f16": [_P, _P],
    "ctrlora_layernorm_f16": [_P, _L, _P, _L, _I, _I, _P, _P, _F, _P],
    "ctrlora_layernorm_grouped_f16": [_P, _L, _P, _L, _I, _I, _P, _P, _P, _P, _I, _F, _P],
    "ctrlora_attention_f16": [_P, _L, _P, _L, _P, _I, _P, _L, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_attention_bwd_f16": [_P, _L, _P, _L, _P, _L, _P, _L, _P, _L, _P, _P, _P, _L, _P, _L, _P, _L, _I, _I, _I, _I, _I, _P],
    "ctrlora_nchw_f32_to_nhwc_f16": [_P, _P, _I, _I, _I, _I, _P],
    "ctrlora_nhwc_to_nchw_f32": [_P, _I, _L, _P, _I, _I, _I, _P],
    "ctrlora_timestep_embedding": [_P, _P, _P, _I, _I, _P],
    "ctrlora_timestep_embedding_f32": [_P, _P, _P, _I, _I, _P],
    "ctrlora_small_linear": [_P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P],
    "ctrlora_upsample2x_f16": [_P, _P, _I, _I, _I, _I, _P],
    "ctrlora_im2col_s2_f16": [_P, _P, _I, _I, _I, _I, _P],
    "ctrlora_cast_transpose_f32_to_f16": [_P, _P, _L, _I, _I, _P],
    "ctrlora_transpose_f16": [_P, _P, _L, _I, _I, _P],
    "ctrlora_conv_dgrad_weight_f16": [_P, _P, _I, _I, _I, _P],
    "ctrlora_set_sm_limit": [_I],
    "ctrlora_ddim_update": [_P, _P, _P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _F, _F, _F, _P],
    "ctrlora_wgrad_tn_f16": [_P, _L, _P, _L, _I, _I, _I, _P, _L, _F, _F, _P, _L, _P],
    "ctrlora_groupnorm_bwd_f16": [_P, _P, _P, _P, _L, _F, _P, _L, _F, _P, _L, _P, _P, _P],
    "ctrlora_layernorm_bwd_f16": [_P, _L, _P, _L, _P, _L, _I, _I, _P, _F, _P, _P, _P, _L, _P],
    "ctrlora_geglu_fwd_f16": [_P, _P, _L, _I, _P],
    "ctrlora_geglu_bwd_f16": [_P, _P, _P, _L, _I, _P],
    "ctrlora_colsum": [_P, _I, _L, _L, _I, _F, _P, _P],
    "ctrlora_image_colsum_f16": [_P, _L, _I, _I, _I, _P, _L, _P],
    "ctrlora_upsample2x_bwd_f16": [_P, _P, _I, _I, _I, _I, _P],
    "ctrlora_im2col_s2_bwd_f16": [_P, _P, _I, _I, _I, _I, _P],
    "ctrlora_mse_loss_grad": [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P],
    "ctrlora_adamw_f32": [_P, _P, _P, _P, _L, _F, _F, _F, _F, _F, _I, _F, _P, _P, _P],
    "ctrlora_adamw_begin": [_P, _P, _F, _F, _P, _P, _P],
    "ctrlora_nonfinite_flag_f32": [_P, _L, _P, _P],
    "ctrlora_im2col_3x3_f16": [_P, _P, _I, _I, _I, _I, _P],
    "ctrlora_outer_accum_f32": [_P, _I, _P, _I, _P, _L, _I, _I, _I, _F, _F, _I, _P],
    "ctrlora_copy2d_f32": [_P, _L, _P, _L, _L, _I, _I, _P],
    "ctrlora_silu_bwd_f32": [_P, _P, _P, _L, _P],
    "ctrlora_cast_rows_f32_to_f16": [_P, _L, _P, _L, _I, _P],
    "ctrlora_im2col_s2_pad_f16": [_P, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_softmax_rows_f32_to_f16": [_P, _L, _P, _L, _L, _I, _F, _P],
    "ctrlora_gaussian_sample": [_P, _P, _P, _I, _I, _I, _F, _P],
    "ctrlora_memset_zero": [_P, _L, _P],
    "ctrlora_q_sample": [_P, _P, _P, _P, _P, _P, _I, _I, _P],
    "ctrlora_ddim_encode_update": [_P, _P, _P, _P, _I, _F, _F, _F, _P],
    "ctrlora_dpm_multistep_update": [_P, _P, _P, _P, _P, _P, _I, _F, _F, _F, _F, _F, _F, _F, _P],
    "ctrlora_plms_update": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _F, _F, _F, _F, _F, _P],
    "ctrlora_weighted_sum_f16": [_P, _P, _I, _P, _L, _P],
    "ctrlora_causal_attention_f16": [_P, _L, _P, _L, _P, _I, _P, _L, _I, _I, _I, _I, _P],
    "ctrlora_clip_embed": [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_quick_gelu_f16": [_P, _L, _P],
    "ctrlora_layernorm_rows": [_P, _I, _L, _P, _I, _L, _I, _I, _P, _P, _F, _P],
    "ctrlora_clip_patch_gather": [_P, _I, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_clip_vision_embed": [_P, _L, _P, _P, _P, _I, _I, _I, _P],
    "ctrlora_patch_gather_hw": [_P, _I, _P, _I, _I, _I, _I, _I, _I, _P],
    "ctrlora_gelu_f16": [_P, _L, _P],
    "ctrlora_dpm_model_output": [_P, _P, _P, _P, _P, _L, _I, _I, _P, _P],
    "ctrlora_dpm_solver_update": [_P, _P, _P, _P, _P, _L, _I, _P, _P],
    "ctrlora_dpm_threshold": [_P, _P, _I, _L, _L, _L, _F, _F, _P],
    "ctrlora_dpm_adaptive_error": [_P, _P, _P, _P, _I, _L, _F, _F, _P],
    "ctrlora_tap_gather_f16": [_P, _I, _L, _P, _I, _I, _I, _I, _P, _I, _I, _I, _P],
    "ctrlora_tap_gather_act_f16": [_P, _I, _L, _P, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_instance_norm_f16": [_P, _P, _P, _P, _L, _I, _I, _I, _I, _I, _I, _F, _P],
    "ctrlora_lineart_out_f16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "ctrlora_lineart_anime_out_f16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _F, _P],
    "ctrlora_hed_side_pool_f16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "ctrlora_hed_fuse": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "ctrlora_openpose_resample": [_P, _I, _I, _I, _I, _P, _P, _I, _P, _P, _I, _P, _I, _I, _P],
    "ctrlora_openpose_smooth": [_P, _P, _P, _I, _I, _I, _P, _I, _P],
    "ctrlora_openpose_peaks": [_P, _P, _I, _I, _I, _D, _P, _L, _P, _P, _P, _P, _I, _P],
    "ctrlora_openpose_limbs": [_P, _I, _I, _I, _P, _P, _I, _P, _P, _I, _P, _P, _P, _I, _L, _I, _D, _P, _P, _P],
    "ctrlora_depth_to_space_bias": [_P, _P, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_add_relu_f16": [_P, _P, _P, _P, _L, _P],
    "ctrlora_upsample_bilinear2x_f16": [_P, _P, _I, _I, _I, _I, _P],
    "ctrlora_midas_head_out_f16": [_P, _P, _P, _P, _L, _I, _P],
    "ctrlora_midas_maps": [_P, _P, _P, _P, _I, _I, _I, _F, _F, _P],
    "ctrlora_dwconv_f16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_resize_bilinear_f16": [_P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P],
    "ctrlora_adaptive_avg_pool_f16": [_P, _I, _P, _I, _I, _I, _I, _P, _I, _P],
    "ctrlora_seg_output": [_P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P],
    "ctrlora_dwconv_act_f16": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P],
    "ctrlora_upsample_bilinear2x_ld_f16": [_P, _I, _P, _I, _I, _I, _I, _I, _P],
    "ctrlora_mlsd_decode": [_P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P],
    "ctrlora_canny_classify": [_P, _L, _I, _I, _I, _I, _I, _P, _P],
    "ctrlora_canny_hysteresis": [_P, _I, _I, _I, _P, _P, _P],
}


def _declare(lib):
    lib.ctrlora_abi_version.restype = c_int
    lib.ctrlora_last_cuda_error.restype = C.c_char_p
    for name in EXPORTS:
        fn = getattr(lib, name)
        if name not in ("ctrlora_abi_version", "ctrlora_last_cuda_error"):
            fn.restype = c_int
            fn.argtypes = _ARGTYPES[name]


def check(status, what):
    if status != 0:
        err = load().ctrlora_last_cuda_error()
        raise CtrloraError(f"{what} failed: {_STATUS.get(status, status)} ({err.decode() if err else ''})")


# Every symbol include/ctrlora_b200.h declares (tests/test_abi.py checks the two lists agree).
EXPORTS = [
    "ctrlora_abi_version",
    "ctrlora_last_cuda_error",
    "ctrlora_gemm_f16",
    "ctrlora_gemm_f16_simt",
    "ctrlora_groupnorm_f16",
    "ctrlora_layernorm_f16",
    "ctrlora_layernorm_grouped_f16",
    "ctrlora_attention_f16",
    "ctrlora_nchw_f32_to_nhwc_f16",
    "ctrlora_nhwc_to_nchw_f32",
    "ctrlora_timestep_embedding",
    "ctrlora_timestep_embedding_f32",
    "ctrlora_small_linear",
    "ctrlora_upsample2x_f16",
    "ctrlora_im2col_s2_f16",
    "ctrlora_cast_transpose_f32_to_f16",
    "ctrlora_transpose_f16",
    "ctrlora_conv_dgrad_weight_f16",
    "ctrlora_set_sm_limit",
    "ctrlora_ddim_update",
    "ctrlora_wgrad_tn_f16",
    "ctrlora_attention_bwd_f16",
    "ctrlora_groupnorm_bwd_f16",
    "ctrlora_layernorm_bwd_f16",
    "ctrlora_geglu_fwd_f16",
    "ctrlora_geglu_bwd_f16",
    "ctrlora_colsum",
    "ctrlora_image_colsum_f16",
    "ctrlora_upsample2x_bwd_f16",
    "ctrlora_im2col_s2_bwd_f16",
    "ctrlora_mse_loss_grad",
    "ctrlora_adamw_f32",
    "ctrlora_adamw_begin",
    "ctrlora_nonfinite_flag_f32",
    "ctrlora_weighted_sum_f16",
    "ctrlora_q_sample",
    "ctrlora_memset_zero",
    "ctrlora_im2col_s2_pad_f16",
    "ctrlora_softmax_rows_f32_to_f16",
    "ctrlora_gaussian_sample",
    "ctrlora_im2col_3x3_f16",
    "ctrlora_outer_accum_f32",
    "ctrlora_copy2d_f32",
    "ctrlora_silu_bwd_f32",
    "ctrlora_cast_rows_f32_to_f16",
    "ctrlora_ddim_encode_update",
    "ctrlora_dpm_multistep_update",
    "ctrlora_plms_update",
    "ctrlora_causal_attention_f16",
    "ctrlora_clip_embed",
    "ctrlora_quick_gelu_f16",
    "ctrlora_layernorm_rows",
    "ctrlora_clip_patch_gather",
    "ctrlora_clip_vision_embed",
    "ctrlora_patch_gather_hw",
    "ctrlora_gelu_f16",
    "ctrlora_dpm_model_output",
    "ctrlora_dpm_solver_update",
    "ctrlora_dpm_threshold",
    "ctrlora_dpm_adaptive_error",
    "ctrlora_tap_gather_f16",
    "ctrlora_tap_gather_act_f16",
    "ctrlora_instance_norm_f16",
    "ctrlora_lineart_out_f16",
    "ctrlora_lineart_anime_out_f16",
    "ctrlora_hed_side_pool_f16",
    "ctrlora_hed_fuse",
    "ctrlora_openpose_resample",
    "ctrlora_openpose_smooth",
    "ctrlora_openpose_peaks",
    "ctrlora_openpose_limbs",
    "ctrlora_depth_to_space_bias",
    "ctrlora_add_relu_f16",
    "ctrlora_upsample_bilinear2x_f16",
    "ctrlora_midas_head_out_f16",
    "ctrlora_midas_maps",
    "ctrlora_dwconv_f16",
    "ctrlora_resize_bilinear_f16",
    "ctrlora_adaptive_avg_pool_f16",
    "ctrlora_seg_output",
    "ctrlora_dwconv_act_f16",
    "ctrlora_upsample_bilinear2x_ld_f16",
    "ctrlora_mlsd_decode",
    "ctrlora_canny_classify",
    "ctrlora_canny_hysteresis",
]
