"""ctypes loader for libmagma_b200.so (the C ABI declared in include/magma_b200.h).

There is deliberately no fallback: if the shared library is missing or the device is not sm_90 every
compute entry point raises. PyTorch is used only for device memory and streams.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmagma_b200.so")

_lib = None
_configured = None  # the handle lib() last configured


class MB200Error(RuntimeError):
    pass


class Operand(ctypes.Structure):
    _fields_ = [
        ("ptr", ctypes.c_void_p),
        ("ld", ctypes.c_int64),
        ("bs0", ctypes.c_int64),
        ("bs1", ctypes.c_int64),
        ("mn_major", ctypes.c_int32),
        ("static_data", ctypes.c_int32),
    ]


class GemmArgs(ctypes.Structure):
    _fields_ = [
        ("M", ctypes.c_int32),
        ("N", ctypes.c_int32),
        ("K", ctypes.c_int32),
        ("nb0", ctypes.c_int32),
        ("nb1", ctypes.c_int32),
        ("c_dtype", ctypes.c_int32),
        ("A", Operand),
        ("B", Operand),
        ("C", ctypes.c_void_p),
        ("ldc", ctypes.c_int64),
        ("c_bs0", ctypes.c_int64),
        ("c_bs1", ctypes.c_int64),
        ("alpha", ctypes.c_float),
        ("act", ctypes.c_int32),
        ("dact", ctypes.c_int32),
        ("accumulate", ctypes.c_int32),
        ("bias", ctypes.c_void_p),
        ("aux_out", ctypes.c_void_p),
        ("aux_in", ctypes.c_void_p),
        ("res1", ctypes.c_void_p),
        ("res2", ctypes.c_void_p),
        ("ld_res", ctypes.c_int64),
        ("force_bn", ctypes.c_int32),
        ("generic_epilogue", ctypes.c_int32),
        ("rope_mode", ctypes.c_int32),
        ("rope_tab", ctypes.c_void_p),
        ("rope_S", ctypes.c_int32),
        ("rope_hd", ctypes.c_int32),
        ("rope_rot", ctypes.c_int32),
        ("rope_ncols", ctypes.c_int32),
        ("splitk_ws", ctypes.c_void_p),
        ("splitk_ws_bytes", ctypes.c_int64),
    ]


def lib():
    """Load (once) and return the ctypes handle, configured with SIGNATURES. Raises MB200Error when the library is not
    built. A handle installed in `_lib` from outside (the CPU emulation libraries of the tests) is configured the first
    time it is returned."""
    global _lib, _configured
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MB200Error(
                f"{LIB_PATH} not found: build it with `python -m magma_b200.build` "
                "(magma_b200 has no CPU / eager fallback)"
            )
        _lib = ctypes.CDLL(LIB_PATH)
    if _lib is not _configured:
        _configured = configure(_lib)
    return _lib


def configure(L):
    """Give every entry point of SIGNATURES that the handle L exports its restype and argtypes, so ctypes converts
    plain Python values and rejects a wrong argument count or type before the call. Returns L."""
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = restype, argtypes
    return L


def check(rc):
    if rc != 0:
        raise MB200Error(f"magma_b200 error {rc}: {lib().mb200_last_error().decode()}")


# ---- model-level runtime structs (include/magma_b200.h) ----
class VitLayerC(ctypes.Structure):
    _fields_ = [
        (n, ctypes.c_void_p)
        for n in (
            "ln1_g", "ln1_b", "w_qkv", "b_qkv", "w_out", "b_out", "ln2_g", "ln2_b", "w_fc", "b_fc", "w_proj", "b_proj",
        )
    ]


class VitModelC(ctypes.Structure):
    _fields_ = [
        ("n_layer", ctypes.c_int32),
        ("width", ctypes.c_int32),
        ("n_head", ctypes.c_int32),
        ("patch", ctypes.c_int32),
        ("image", ctypes.c_int32),
        ("mlp", ctypes.c_int32),
        ("out_dim", ctypes.c_int32),
        ("_pad", ctypes.c_int32),
        ("w_conv", ctypes.c_void_p),
        ("ld_conv", ctypes.c_int64),
        ("cls", ctypes.c_void_p),
        ("pos", ctypes.c_void_p),
        ("ln_pre_g", ctypes.c_void_p),
        ("ln_pre_b", ctypes.c_void_p),
        ("ln_post_g", ctypes.c_void_p),
        ("ln_post_b", ctypes.c_void_p),
        ("proj_t", ctypes.c_void_p),
        ("layers", ctypes.POINTER(VitLayerC)),
    ]


class AdapterExC(ctypes.Structure):
    """mb200_adapter_ex: adapter bottleneck with the optional leading LayerNorm and the learnable scale."""
    _fields_ = [(n, ctypes.c_void_p) for n in ("wd", "bd", "wu", "bu", "ln_g", "ln_b", "scale", "g_wd", "g_bd", "g_wu",
                                               "g_bu", "g_ln_g", "g_ln_b", "g_scale")]


class GptjLayerExC(ctypes.Structure):
    _fields_ = [
        (n, ctypes.c_void_p)
        for n in ("ln1_g", "ln1_b", "w_qkv", "w_out", "w_fc_in", "b_fc_in", "w_fc_out", "b_fc_out")
    ] + [("mlp_ad", AdapterExC), ("attn_ad", AdapterExC)]


class GptjLayerGradsC(ctypes.Structure):
    """mb200_gptj_layer_grads: fp32 gradients of one block's own weights (NULL = frozen)."""
    _fields_ = [(n, ctypes.c_void_p) for n in ("ln1_g", "ln1_b", "w_qkv", "w_out", "w_fc_in", "b_fc_in", "w_fc_out",
                                               "b_fc_out")]


class GptjLmGradsC(ctypes.Structure):
    """mb200_gptj_lm_grads."""
    _fields_ = [("layers", ctypes.POINTER(GptjLayerGradsC))] + [
        (n, ctypes.c_void_p) for n in ("lnf_g", "lnf_b", "w_lm", "b_lm")]


class GptjModelExC(ctypes.Structure):
    """mb200_gptj_model_ex (include/magma_b200.h)."""
    _fields_ = [
        ("n_layer", ctypes.c_int32),
        ("d", ctypes.c_int32),
        ("n_head", ctypes.c_int32),
        ("rotary_dim", ctypes.c_int32),
        ("vocab", ctypes.c_int32),
        ("d_ff", ctypes.c_int32),
        ("mlp_adapter", ctypes.c_int32),
        ("mlp_adapter_r", ctypes.c_int32),
        ("attn_adapter", ctypes.c_int32),
        ("attn_adapter_r", ctypes.c_int32),
        ("ln_eps", ctypes.c_float),
        ("adapter_act", ctypes.c_int32),
        ("layers", ctypes.POINTER(GptjLayerExC)),
        ("lnf_g", ctypes.c_void_p),
        ("lnf_b", ctypes.c_void_p),
        ("w_lm", ctypes.c_void_p),
        ("b_lm", ctypes.c_void_p),
        ("lm_grads", ctypes.POINTER(GptjLmGradsC)),
    ]


class VitLayerGradsC(ctypes.Structure):
    """mb200_vit_layer_grads: fp32 gradient pointers, same field order as VitLayerC."""
    _fields_ = list(VitLayerC._fields_)


class VitGradsC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("w_conv", "cls", "pos", "ln_pre_g", "ln_pre_b", "ln_post_g",
                                               "ln_post_b", "proj")] + [("layers", ctypes.POINTER(VitLayerGradsC))]


# ---- (restype, argtypes) of every entry point, in the order of include/magma_b200.h ----
# int32_t / int -> c_int32, int64_t -> c_int64, uint64_t -> c_uint64, size_t -> c_size_t, float -> c_float,
# long long -> c_longlong, const char* (return) -> c_char_p, const mb200_<struct>* -> POINTER(<its mirror above>),
# void* const* -> POINTER(c_void_p), every other data pointer and the stream -> c_void_p.
_i32, _i64, _u64, _f32 = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64, ctypes.c_float
_sz, _vp = ctypes.c_size_t, ctypes.c_void_p
_VPP = ctypes.POINTER(_vp)
_GEMM, _VIT, _VITG, _GPTJ = (ctypes.POINTER(t) for t in (GemmArgs, VitModelC, VitGradsC, GptjModelExC))

SIGNATURES = {
    "mb200_version": (_i32, []),
    "mb200_last_error": (ctypes.c_char_p, []),
    "mb200_check_device": (_i32, []),
    "mb200_set_gemm_sm_limit": (_i32, [_i32]),
    "mb200_set_optimizer_grid": (_i32, [_i32]),
    "mb200_launch_count": (ctypes.c_longlong, []),
    "mb200_prof_enable": (_i32, [_i32]),
    "mb200_prof_read": (_i32, [_vp, _vp, _vp, _vp]),
    "mb200_gemm": (_i32, [_GEMM, _vp]),
    "mb200_gemm_last_plan": (_i32, [_vp, _vp]),
    "mb200_layernorm_fwd": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _i32, _i32, _f32, _vp]),
    "mb200_layernorm_bwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _i32, _i32, _vp]),
    "mb200_layernorm_param_grad": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "mb200_layernorm_param_grad_rows": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "mb200_rope": (_i32, [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_rope_table": (_i32, [_vp, _i32, _i32, _i32, _vp]),
    "mb200_softmax_fwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _f32, _i32, _i32, _vp]),
    "mb200_softmax_bwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _f32, _vp]),
    "mb200_build_labels": (_i32, [_vp, _i64, _vp, _i32, _i32, _i32, _i64, _vp]),
    "mb200_embed_assemble": (_i32, [_vp, _i64, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _i32, _vp]),
    "mb200_embed_gather": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "mb200_embed_grad": (_i32, [_vp, _i64, _vp, _i64, _i64, _i32, _i32, _vp, _i32, _i32, _i32, _vp]),
    "mb200_cross_entropy": (_i32, [_vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _vp]),
    "mb200_colsum": (_i32, [_vp, _i64, _i32, _i32, _vp, _i32, _vp]),
    "mb200_dropout_fwd": (_i32, [_vp, _vp, _vp, _i64, _f32, _u64, _vp]),
    "mb200_dropout_apply": (_i32, [_vp, _vp, _vp, _i64, _f32, _vp]),
    "mb200_patchify": (_i32, [_vp, _vp, _i64, _i32, _i32, _i32, _vp]),
    "mb200_vit_assemble": (_i32, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "mb200_nchw_to_nhwc8": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "mb200_im2col3x3": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_avgpool_nhwc": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_col_moments": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _vp, _vp, _vp]),
    "mb200_channel_affine": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _i64, _i32, _vp]),
    "mb200_bn_finalize_fwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _f32, _f32, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _vp]),
    "mb200_bn_bwd_coeffs": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _vp]),
    "mb200_col2im3x3": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_avgpool_nhwc_bwd": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_argmax": (_i32, [_vp, _i64, _i32, _i32, _vp, _vp]),
    "mb200_sample": (_i32, [_vp, _i32, _i64, _i32, _i32, _f32, _i32, _f32, _u64, _u64, _vp, _vp, _vp]),
    "mb200_add": (_i32, [_vp, _vp, _vp, _vp, _i64, _vp]),
    "mb200_logits_grad_combine": (_i32, [_vp, _i64, _vp, _i64, _vp, _i32, _i32, _f32, _vp]),
    "mb200_peer_reduce_bcast": (_i32, [ctypes.POINTER(_vp), _i32, _i64, _i64, _i32, _vp]),
    "mb200_sumsq": (_i32, [_vp, _i64, _vp, _vp]),
    "mb200_adamw_step": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _f32, _f32, _vp, _f32, _i32,
                                _i32, _vp]),
    "mb200_cast_f32_to_bf16": (_i32, [_vp, _vp, _i64, _vp]),
    "mb200_cast_bf16_to_f32": (_i32, [_vp, _vp, _i64, _vp]),
    "mb200_vit_workspace_bytes": (_sz, [_VIT, _i32]),
    "mb200_vit_forward": (_i32, [_VIT, _vp, _vp, _i32, _vp, _sz, _vp]),
    "mb200_vit_train_workspace_bytes": (_sz, [_VIT, _i32]),
    "mb200_vit_forward_train": (_i32, [_VIT, _vp, _vp, _i32, _vp, _sz, _vp]),
    "mb200_vit_backward": (_i32, [_VIT, _VITG, _vp, _i32, _i32, _vp, _sz, _vp]),
    "mb200_quick_gelu_bwd": (_i32, [_vp, _vp, _vp, _i64, _vp]),
    "mb200_gptj_sched_workspace_bytes": (_sz, [_GPTJ, _i32, _i32]),
    "mb200_gptj_sched_forward": (_i32, [_GPTJ, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_backward": (_i32, [_GPTJ, _vp, _f32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_backward_range": (_i32, [_GPTJ, _vp, _f32, _i32, _i32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_recompute_workspace_bytes": (_sz, [_GPTJ, _i32, _i32]),
    "mb200_gptj_sched_forward_recompute": (_i32, [_GPTJ, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_backward_range_recompute": (_i32, [_GPTJ, _vp, _f32, _i32, _i32, _i32, _i32, _i32, _vp, _sz,
                                                         _vp]),
    "mb200_gptj_sched_hidden_states": (_i32, [_GPTJ, _VPP, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_hidden_states_recompute": (_i32, [_GPTJ, _VPP, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_backward_range_hidden": (_i32, [_GPTJ, _vp, _VPP, _f32, _i32, _i32, _i32, _i32, _i32, _vp, _sz,
                                                      _vp]),
    "mb200_gptj_sched_backward_range_hidden_recompute": (_i32, [_GPTJ, _vp, _VPP, _f32, _i32, _i32, _i32, _i32, _i32,
                                                                _vp, _sz, _vp]),
    "mb200_gptj_sched_forward_attn": (_i32, [_GPTJ, _vp, _vp, _vp, _i64, _vp, _VPP, _i64, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_forward_attn_recompute": (_i32, [_GPTJ, _vp, _vp, _vp, _i64, _vp, _VPP, _i64, _i32, _i32, _vp, _sz,
                                                       _vp]),
    "mb200_gptj_sched_backward_range_attn": (_i32, [_GPTJ, _vp, _VPP, _VPP, _i64, _f32, _i32, _i32, _i32, _i32, _i32, _vp,
                                                    _sz, _vp]),
    "mb200_gptj_sched_backward_range_attn_recompute": (_i32, [_GPTJ, _vp, _VPP, _VPP, _i64, _f32, _i32, _i32, _i32, _i32,
                                                              _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_backward_range_logits": (_i32, [_GPTJ, _vp, _VPP, _VPP, _i64, _vp, _i64, _vp, _f32, _i32, _i32,
                                                      _i32, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_backward_range_logits_recompute": (_i32, [_GPTJ, _vp, _VPP, _VPP, _i64, _vp, _i64, _vp, _f32, _i32,
                                                                _i32, _i32, _i32, _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_infer_workspace_bytes": (_sz, [_GPTJ, _i32, _i32, _i32]),
    "mb200_gptj_sched_infer": (_i32, [_GPTJ, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _sz,
                                      _vp]),
    "mb200_gptj_sched_infer_hidden": (_i32, [_GPTJ, _vp, _vp, _i64, _i32, _vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32,
                                             _vp, _sz, _vp]),
    "mb200_gptj_sched_infer_attn": (_i32, [_GPTJ, _vp, _vp, _i64, _i32, _vp, _i64, _VPP, _i64, _vp, _vp, _i32, _i32, _i32,
                                           _i32, _vp, _sz, _vp]),
    "mb200_gptj_sched_decode_step": (_i32, [_GPTJ, _vp, _vp, _i64, _vp, _vp, _i32, _vp, _i32, _vp, _sz, _vp]),
    "mb200_decode_embed": (_i32, [_vp, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "mb200_decode_advance": (_i32, [_vp, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _vp]),
    "mb200_sample_dev": (_i32, [_vp, _i32, _i64, _i32, _i32, _f32, _i32, _f32, _u64, _vp, _i32, _vp, _vp, _vp]),
    "mb200_rope_table_dev": (_i32, [_vp, _i32, _i32, _vp, _vp]),
    "mb200_attn_decode_dev": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "mb200_scale_add": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "mb200_dot": (_i32, [_vp, _vp, _i64, _vp, _i32, _vp]),
    "mb200_attn_fwd_tile": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _vp]),
    "mb200_attn_bwd_tile": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_attn_bwd_tile_dp": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32,
                                      _i32, _vp]),
    "mb200_attn_fwd_flash": (_i32, [_vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64, _vp, _i64, _vp,
                                    _i64, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_attn_decode": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_attn_decode_probs": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    "mb200_kv_append": (_i32, [_vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
}

EXPORTED_SYMBOLS = list(SIGNATURES)
