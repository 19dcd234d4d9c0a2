"""ctypes loader for libmagma_b200.so (the C ABI declared in include/magma_b200.h).

There is deliberately no fallback: if the shared library is missing or the device is not sm_90 every
compute entry point raises. PyTorch is used only for device memory and streams.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmagma_b200.so")

_lib = None


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
    """Load (once) and return the ctypes handle. Raises MB200Error when the library is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MB200Error(
                f"{LIB_PATH} not found: build it with `python -m magma_b200.build` "
                "(magma_b200 has no CPU / eager fallback)"
            )
        L = ctypes.CDLL(LIB_PATH)
        L.mb200_last_error.restype = ctypes.c_char_p
        L.mb200_version.restype = ctypes.c_int
        _setup_signatures(L)
        _lib = L
    return _lib


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
    ]


class VitLayerGradsC(ctypes.Structure):
    """mb200_vit_layer_grads: fp32 gradient pointers, same field order as VitLayerC."""
    _fields_ = list(VitLayerC._fields_)


class VitGradsC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("w_conv", "cls", "pos", "ln_pre_g", "ln_pre_b", "ln_post_g",
                                               "ln_post_b", "proj")] + [("layers", ctypes.POINTER(VitLayerGradsC))]


def _setup_signatures(L):
    L.mb200_vit_workspace_bytes.restype = ctypes.c_size_t
    L.mb200_vit_train_workspace_bytes.restype = ctypes.c_size_t
    L.mb200_gptj_sched_workspace_bytes.restype = ctypes.c_size_t
    L.mb200_gptj_sched_infer_workspace_bytes.restype = ctypes.c_size_t
    L.mb200_gptj_sched_recompute_workspace_bytes.restype = ctypes.c_size_t
    L.mb200_launch_count.restype = ctypes.c_longlong


EXPORTED_SYMBOLS = [
    "mb200_version", "mb200_last_error", "mb200_check_device", "mb200_gemm", "mb200_gemm_last_plan",
    "mb200_launch_count", "mb200_prof_enable", "mb200_prof_read",
    "mb200_layernorm_fwd", "mb200_layernorm_bwd", "mb200_layernorm_param_grad", "mb200_rope", "mb200_rope_table",
    "mb200_softmax_fwd", "mb200_softmax_bwd", "mb200_build_labels", "mb200_embed_assemble", "mb200_embed_gather",
    "mb200_cross_entropy", "mb200_colsum", "mb200_dropout_fwd", "mb200_dropout_apply", "mb200_patchify",
    "mb200_nchw_to_nhwc8", "mb200_im2col3x3", "mb200_avgpool_nhwc",
    "mb200_vit_assemble", "mb200_argmax", "mb200_sample", "mb200_add", "mb200_peer_reduce_bcast", "mb200_sumsq", "mb200_adamw_step",
    "mb200_cast_f32_to_bf16", "mb200_cast_bf16_to_f32",
    "mb200_vit_workspace_bytes", "mb200_vit_forward", "mb200_attn_decode", "mb200_attn_fwd_tile", "mb200_attn_fwd_flash",
    "mb200_attn_bwd_tile",
    "mb200_vit_train_workspace_bytes", "mb200_vit_forward_train", "mb200_vit_backward", "mb200_quick_gelu_bwd",
    "mb200_layernorm_param_grad_rows", "mb200_set_gemm_sm_limit", "mb200_set_optimizer_grid", "mb200_scale_add", "mb200_dot",
    "mb200_gptj_sched_workspace_bytes", "mb200_gptj_sched_forward", "mb200_gptj_sched_backward",
    "mb200_col_moments", "mb200_channel_affine", "mb200_col2im3x3", "mb200_avgpool_nhwc_bwd",
    "mb200_kv_append", "mb200_gptj_sched_infer_workspace_bytes", "mb200_gptj_sched_infer",
    "mb200_gptj_sched_backward_range", "mb200_bn_finalize_fwd", "mb200_bn_bwd_coeffs",
    "mb200_gptj_sched_decode_step", "mb200_decode_embed", "mb200_decode_advance", "mb200_rope_table_dev",
    "mb200_attn_decode_dev", "mb200_gptj_sched_recompute_workspace_bytes", "mb200_gptj_sched_forward_recompute",
    "mb200_gptj_sched_backward_range_recompute",
]
