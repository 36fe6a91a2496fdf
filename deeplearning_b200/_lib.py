"""ctypes binding of libb200cls.so (the C-ABI boundary declared in include/b200cls.h).

There is no fallback: if the shared library is missing, or a call fails, a RuntimeError is raised.
Build it with ``python -c "import __graft_entry__ as g; g.build()"`` or ``make -C deeplearning_b200/csrc``.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# (B200_LIB: an alternate build of the same ABI, for A/B experiments)
LIB_PATH = os.environ.get("B200_LIB") or os.path.join(_HERE, "lib", "libb200cls.so")

_lib = None

_P = c_void_p
_I = c_int
_L = c_longlong
_F = c_float
_D = c_double

class View(ctypes.Structure):
    """b200_view_t"""
    _fields_ = [("base", c_void_p), ("dim", c_longlong * 3), ("stride", c_longlong * 3)]


class GemmArgs(ctypes.Structure):
    """b200_gemm_args_t"""
    _fields_ = [("w", c_void_p), ("N", c_int), ("K", c_int), ("bias", c_void_p), ("colscale", c_void_p), ("act", c_int),
                ("out_f32", c_int),
                ("residual", ctypes.POINTER(View)), ("residual_f32", c_int), ("aux_out", ctypes.POINTER(View)),
                ("aux_in", ctypes.POINTER(View)), ("stats", c_void_p), ("rowscale", c_void_p), ("rows_per_sample", c_int)]


class BnMask(ctypes.Structure):
    """b200_bn_mask_t"""
    _fields_ = [("x_raw", c_void_p), ("scale", c_void_p), ("shift", c_void_p), ("stats", c_void_p)]



# name -> (restype, argtypes); must list every symbol of include/b200cls.h (tests/test_abi.py checks this).
SIGNATURES = {
    "b200_last_error": (c_char_p, []),
    "b200_abi_version": (_I, []),
    "b200_sm_count": (_I, []),
    "b200_launch_count": (ctypes.c_ulonglong, []),
    "b200_conv2d_fwd": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _I, _P, _P, _L, _P, _P, _P]),
    "b200_conv2d_fwd_stats_rows": (_I, [_I, _I, _I, _I, _I, _I]),
    "b200_conv2d_dgrad": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, ctypes.POINTER(BnMask), _P]),
    "b200_conv2d_wgrad": (_I, [_P, _P, _P, _P, c_size_t, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "b200_conv2d_wgrad_workspace_bytes": (c_size_t, [_I, _I, _I, _I, _I, _I, _I]),
    "b200_reduce_scratch_bytes": (c_size_t, [_I, _I]),
    "b200_gemm_ex": (_I, [ctypes.POINTER(View), ctypes.POINTER(View), ctypes.POINTER(GemmArgs), _P]),
    "b200_layernorm_fwd": (_I, [_P, _I, _P, _P, _P, _I, _P, _P, _L, _I, _F, _P]),
    "b200_layernorm_bwd_blocks": (_I, [_L, _I]),
    "b200_layernorm_bwd": (_I, [_P, _P, _I, _P, _P, _P, _P, _P, _I, _P, _L, _I, _P]),
    "b200_patchify_nchw": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "b200_cls_row": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "b200_batch_rowsum": (_I, [_P, _I, _L, _I, _I, _P, _I, _P]),
    "b200_copy_rows": (_I, [_P, _L, _P, _L, _L, _L, _P]),
    "b200_colsum_partial_slices": (_I, [_L]),
    "b200_colsum_partial": (_I, [_P, _L, _L, _I, _P, _P]),
    "b200_attention_fwd": (_I, [_P, _P, _P, _I, _I, _I, _F, _P]),
    "b200_attention_bwd": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _P]),
    "b200_conv2d_wgrad_splits": (_I, [_I, _I, _I, _I, _I, _I, _I]),
    "b200_conv2d_grouped_fwd": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _I, _P, _P, _P]),
    "b200_conv2d_grouped_fwd_stats_rows": (_I, [_I, _I, _I, _I, _I, _I, _I]),
    "b200_conv2d_grouped_dgrad": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, ctypes.POINTER(BnMask), _P]),
    "b200_conv2d_grouped_wgrad": (_I, [_P, _P, _P, _P, c_size_t, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_conv2d_grouped_wgrad_workspace_bytes": (c_size_t, [_I, _I, _I, _I, _I, _I, _I]),
    "b200_dwconv7_pack": (_I, [_P, _P, _I, _P]),
    "b200_dwconv7": (_I, [_P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "b200_dwconv7_wgrad_workspace_bytes": (c_size_t, [_I, _I, _I, _I]),
    "b200_dwconv7_wgrad": (_I, [_P, _P, _P, _P, c_size_t, _I, _I, _I, _I, _I, _P]),
    "b200_avgpool_any": (_I, [_P, _I, _P, _I, _I, _I, _P]),
    "b200_colsum_prod_partial": (_I, [_P, _P, _L, _L, _I, _P, _P]),
    "b200_layerscale_grads": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _P]),
    "b200_conv2d_fwd_f32": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    "b200_adamw_tick": (_I, [_P, _F, _F, _P]),
    "b200_adamw": (_I, [_P, _P, _P, _P, _P, _L, _P, _F, _F, _F, _F, _P, _P]),
    "b200_grad_clip_blocks": (_I, []),
    "b200_grad_clip_coef": (_I, [_P, _L, _F, _F, _P, _P, _P]),
    "b200_window_attention_fwd": (_I, [_P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _F, _P]),
    "b200_window_attention_bwd": (_I, [_P, _P, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P]),
    "b200_window_bias_gather": (_I, [_P, _P, _P, _I, _P, _I, _P]),
    "b200_window_bias_scatter": (_I, [_P, _P, _P, _I, _P]),
    "b200_window_partition": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_window_merge": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_patch_merge_ln_fwd": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "b200_patch_merge_ln_bwd_blocks": (_I, [_L]),
    "b200_patch_merge_ln_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "b200_bn_finalize": (_I, [_P, _I, _I, _D, _P, _P, _F, _F, _P, _P, _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "b200_bn_eval_coeffs": (_I, [_I, _P, _P, _P, _P, _F, _P, _P, _P]),
    "b200_bn_apply": (_I, [_P, _P, _P, _P, _P, _L, _I, _I, _P]),
    "b200_bn_bwd_reduce": (_I, [_P, _P, _P, _P, _P, _P, _I, _L, _I, _P, _P]),
    "b200_bn_bwd_blocks": (_I, [_L, _I]),
    "b200_bn_bwd_finalize": (_I, [_P, _I, _I, _D, _P, _P, _I, _P, _P, _P, _P, _P, c_size_t, _P]),
    "b200_bn_bwd_apply": (_I, [_P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I, _L, _I, _P]),
    "b200_bn_relu_maxpool_fwd": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "b200_maxpool_bwd": (_I, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "b200_avgpool_fwd": (_I, [_P, _P, _I, _I, _I, _P]),
    "b200_avgpool_bwd": (_I, [_P, _P, _I, _I, _I, _P]),
    "b200_softmax_xent": (_I, [_P, _L, _P, _I, _I, _F, _P, _P, _L, _P, _P]),
    "b200_softmax_xent_soft": (_I, [_P, _L, _P, _P, _L, _F, _I, _I, _F, _P, _P, _L, _P, _P]),
    "b200_mean": (_I, [_P, _I, _P, _P]),
    "b200_colsum_bf16": (_I, [_P, _L, _L, _I, _P, _I, _P]),
    "b200_pack_weight": (_I, [_P, _P, _I, _I, _I, _I, _L, _P]),
    "b200_pack_weights_multi": (_I, [_P, _I, _I, _P]),
    "b200_cast_f32_to_bf16": (_I, [_P, _P, _L, _P]),
    "b200_cast_bf16_to_f32": (_I, [_P, _P, _L, _P]),
    "b200_im2col_nchw": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_stem_wgrad_relayout": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "b200_stem_s2d": (_I, [_P, _P, _I, _I, _I, _P]),
    "b200_stem_s2d_u8": (_I, [_P, _P, _I, _I, _I, ctypes.POINTER(c_float), ctypes.POINTER(c_float), _P]),
    "b200_normalize_u8_nhwc": (_I, [_P, _P, _I, _I, _I, ctypes.POINTER(c_float), ctypes.POINTER(c_float), _P]),
    "b200_stem_s2d_conv_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "b200_stem_s2d_conv_wgrad_workspace_bytes": (c_size_t, [_I, _I, _I]),
    "b200_stem_s2d_conv_wgrad": (_I, [_P, _P, _P, _P, c_size_t, _I, _I, _I, _P]),
    "b200_stem_s2d_wgrad_relayout": (_I, [_P, _P, _I, _P]),
    "b200_bn_gram_stats": (_I, [_P, _P, _P, _I, _I, _D, _P, _P, _F, _F, _P, _P, _P, _P, _P, _P, _P, _P]),
    "b200_conv1x1_bn_act_fwd": (_I, [_P, _P, _P, _P, _P, _P, _L, _I, _I, _I, _P]),
    "b200_conv1x1_bn_fwd": (_I, [_P, _P, _P, _P, _P, _L, _I, _I, _P]),
    "b200_subsample2": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "b200_add_even_pixels": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "b200_conv1x1_dgrad_masked_stats_rows": (_I, [_L, _I, _I]),
    "b200_conv1x1_dgrad_masked": (_I, [_P, _P, _P, _L, _I, _I, _P, _P, _P, _P]),
    "b200_bn_conv1x1_bwd_scratch_bytes": (c_size_t, [_I, _I]),
    "b200_bn_conv1x1_bwd": (_I, [_P, _I, _P, _P, _P, _P, _P, _I, _I, _D, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, c_size_t, _P, _P]),
    "b200_gemm_dual": (_I, [_P, _I, _P, _I, _P, _P, _P, _L, _I, ctypes.POINTER(BnMask), _P]),
    "b200_rowscale_bf16": (_I, [_P, _P, _P, _L, _L, _P]),
    "b200_tanh_fwd": (_I, [_P, _P, _P, _L, _P]),
    "b200_tanh_bwd": (_I, [_P, _P, _P, _L, _P]),
    "b200_sgd_momentum": (_I, [_P, _P, _P, _L, _F, _P, _F, _F, _F, _I, _P, _P]),
    "b200_se_squeeze": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "b200_se_excite": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "b200_se_apply": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "b200_se_bwd_reduce": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "b200_se_bwd_coeffs": (_I, [_P] * 12 + [_I, _I, _I, _I] + [_P] * 9),
    "b200_se_bwd_apply": (_I, [_P] * 10 + [_I, _I, _I, _P]),
    "b200_repvgg_partial_rows": (_I, [_L, _I]),
    "b200_repvgg_apply": (_I, [_P, _L, _P, _L, _P, _L, _P, _P, _P, _P, _L, _I, _P, _P]),
    "b200_repvgg_bwd_reduce": (_I, [_P, _P, _P, _L, _P, _L, _P, _L, _L, _I, _P, _P]),
    "b200_repvgg_bwd_apply": (_I, [_P, _P, _P, _L, _P, _L, _P, _L] + [_P] * 9 + [_L, _I, _P]),
    "b200_repvgg_fold": (_I, [_P, _P, _P, _P, _P, _P, _F, _P, _P, _P, _P, _F, _P, _P, _P, _P, _F, _I, _I, _I, _P, _P, _P]),
    "b200_dw_partial_rows": (_I, [_L, _I]),
    "b200_dw_fwd": (_I, [_P] * 6 + [_I] * 6 + [_P]),
    "b200_dw_dgrad": (_I, [_P] * 8 + [_I] * 6 + [_P]),
    "b200_dw_wgrad_workspace_bytes": (c_size_t, [_I] * 6),
    "b200_dw_wgrad": (_I, [_P] * 6 + [c_size_t] + [_I] * 6 + [_P]),
    "b200_silu_bn_squeeze": (_I, [_P] * 6 + [_I] * 3 + [_P]),
    "b200_excite_fwd": (_I, [_P] * 7 + [_I] * 3 + [_P]),
    "b200_excite_bwd": (_I, [_P] * 13 + [_I] * 3 + [_P]),
    "b200_gate_apply": (_I, [_P] * 5 + [_I] * 3 + [_P]),
    "b200_gate_reduce": (_I, [_P] * 5 + [_I] * 3 + [_P]),
    "b200_silu_bn_bwd_reduce": (_I, [_P] * 8 + [_I] * 3 + [_P]),
    "b200_tail_apply": (_I, [_P] * 6 + [_I] * 3 + [_P]),
    "b200_tail_bwd_reduce": (_I, [_P] * 5 + [_I] * 3 + [_P]),
    "b200_bn_bwd_apply_dz": (_I, [_P] * 5 + [_L, _I, _P]),
    "b200_vgg_pool_partial_rows": (_I, [_I, _I, _I, _I]),
    "b200_vgg_pool_fwd": (_I, [_P] * 5 + [_I] * 4 + [_P]),
    "b200_vgg_pool_bwd": (_I, [_P] * 8 + [_I] * 4 + [_P]),
    "b200_vgg_avgpool7_fwd": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "b200_vgg_avgpool7_bwd": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "b200_vgg_dropout_fwd": (_I, [_P, _P, _P, _L, _P]),
    "b200_vgg_dropout_bwd": (_I, [_P, _P, _F, _P, _L, _P]),
    "b200_adam": (_I, [_P, _P, _P, _P, _L, _P, _F, _F, _F, _F, _F, _P, _P]),
}


def load():
    """Load (once) and return the ctypes handle; raises if the library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: the CUDA extension is not built (run __graft_entry__.build()); "
            "deeplearning_b200 has no CPU / PyTorch fallback for the hot path"
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    msg = load().b200_last_error()
    return msg.decode() if msg else ""


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {last_error()}")
