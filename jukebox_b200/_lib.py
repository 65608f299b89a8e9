"""ctypes binding of libjkb200.so (the C ABI declared in include/jkb200.h).

There is no fallback: if the shared library is missing this module raises at import of
`lib()` time, and every op that needs the GPU raises when handed a non-CUDA tensor.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libjkb200.so")

JK_MAX_DEPTH = 96
JK_MAX_BATCH = 32
JK_XOUT_STATS_MAX_K = 16        # jkb200.h: the largest top-k jk_xout_stats returns


class PriorConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in
                ("width", "depth", "heads", "n_state", "mlp_width", "n_ctx", "blocks", "bins",
                 "prime_len", "encoder_dims", "max_batch", "add_cond_after")] + \
               [("attn_func", C.c_int32 * JK_MAX_DEPTH)]


class LayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("c_attn_w", "c_attn_b", "c_enc_kv_w", "c_enc_kv_b", "c_proj_w", "c_proj_b",
                 "fc_w", "fc_b", "proj2_w", "proj2_b", "ln0_g", "ln0_b", "ln1_g", "ln1_b")] + \
               [("w_dtype", C.c_int32), ("b_dtype", C.c_int32)]


class PlanInfo(C.Structure):
    _fields_ = [("k_split", C.c_int32), ("units", C.c_int32), ("ring_slots", C.c_int32), ("smem_bytes", C.c_int32),
                ("tile_rows", C.c_int32), ("logits_passes", C.c_int32), ("arena_bytes", C.c_uint64),
                ("stream_stride", C.c_uint64)]


class F32Layer(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("ln0_g", "ln0_b", "ln1_g", "ln1_b", "c_attn_w", "c_attn_b", "c_enc_kv_w", "c_enc_kv_b",
                 "c_proj_w", "c_proj_b", "fc_w", "fc_b", "proj2_w", "proj2_b", "k_cache", "v_cache", "attn_w")] + \
               [("attn_func", C.c_int32)]


class F32Args(C.Structure):
    _fields_ = [(n, C.c_int32) for n in
                ("n", "P", "p0", "width", "n_state", "mlp_width", "heads", "n_ctx", "blocks", "prime_len",
                 "encoder_dims", "depth")] + \
               [("x", C.c_void_p), ("encoder_kv", C.c_void_p), ("work", C.c_void_p)]


class F32GradLayer(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("ln0_g", "ln0_b", "ln1_g", "ln1_b", "c_attn_w", "c_attn_b", "c_enc_kv_w", "c_enc_kv_b",
                 "c_proj_w", "c_proj_b", "fc_w", "fc_b", "proj2_w", "proj2_b")]


class StepArgs(C.Structure):
    _fields_ = [("n_samples", C.c_int32), ("x_in", C.c_void_p), ("tokens", C.c_void_p),
                ("tok_stride", C.c_int64), ("y_cond", C.c_void_p), ("x_cond", C.c_void_p),
                ("x_cond_len", C.c_int64), ("h_out", C.c_void_p), ("logits", C.c_void_p),
                ("logits_bstride", C.c_int64), ("logits_tstride", C.c_int64), ("logit_bias", C.c_void_p),
                ("logit_bias_bstride", C.c_int64), ("logit_bias_tstride", C.c_int64)]


class AttnRecord(C.Structure):
    _fields_ = [("layer", C.c_int32), ("ld", C.c_int32), ("w", C.c_void_p)]


class ActCapture(C.Structure):
    _fields_ = [("layer", C.c_int32), ("t0", C.c_int32), ("t1", C.c_int32), ("pool", C.c_int32),
                ("add_x_cond", C.c_int32), ("out", C.c_void_p)]


class PrefillArgs(C.Structure):
    _fields_ = [("n_samples", C.c_int32), ("n_positions", C.c_int32), ("tokens", C.c_void_p),
                ("tok_stride", C.c_int64), ("y_cond", C.c_void_p), ("x_cond", C.c_void_p),
                ("x_cond_len", C.c_int64), ("h_out", C.c_void_p), ("record", C.POINTER(AttnRecord)),
                ("n_record", C.c_int32), ("n_layers", C.c_int32), ("capture", C.POINTER(ActCapture)),
                ("n_capture", C.c_int32)]


class PrefillAttnArgs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("qkv", "k_cache", "v_cache", "out", "w")] + \
               [(n, C.c_int32) for n in
                ("ld", "n", "P", "heads", "dh", "dh_pad", "attn_func", "bc", "prime", "enc_rows", "route", "q_offset",
                 "cache_rows", "blocks")]


class PrefillAttnRoute(C.Structure):
    _fields_ = [("tensor_cores", C.c_int32), ("tile_dh", C.c_int32), ("stage_bytes", C.c_int32)]


class SelectPlanInfo(C.Structure):
    _fields_ = [("n_copies", C.c_int32), ("n_stash", C.c_int32), ("stash", C.c_int32 * JK_MAX_BATCH),
                ("row_bytes", C.c_uint64), ("workspace_bytes", C.c_uint64), ("bytes_moved", C.c_uint64)]


class ConvArgs(C.Structure):
    _fields_ = [("inp", C.c_void_p), ("t_in", C.c_int64), ("c_in", C.c_int32),
                ("out", C.c_void_p), ("t_out", C.c_int64), ("c_out", C.c_int32),
                ("w", C.c_void_p), ("bias", C.c_void_p), ("res", C.c_void_p),
                ("n_taps", C.c_int32), ("tap_off", C.c_int32 * 4), ("in_stride", C.c_int32),
                ("out_stride", C.c_int32), ("out_offset", C.c_int32), ("relu_in", C.c_int32),
                ("scale", C.c_float), ("n", C.c_int32), ("tensor_cores", C.c_int32)]


# every symbol include/jkb200.h declares: name -> (restype, argtypes)
_P, _I, _L, _F = C.c_void_p, C.c_int, C.c_int64, C.c_float
SIGNATURES = {
    "jk_last_error": (C.c_char_p, []),
    "jk_version": (_I, []),
    "jk_device_sm_count": (_I, [C.POINTER(C.c_int)]),
    "jk_prior_plan": (_I, [C.POINTER(PriorConfig), _I, C.POINTER(PlanInfo), _P, C.c_size_t]),
    "jk_prior_arena_bytes": (_I, [C.POINTER(PriorConfig), C.POINTER(C.c_size_t)]),
    "jk_prior_create": (_I, [C.POINTER(PriorConfig), _P, C.c_size_t, C.POINTER(_P), _P]),
    "jk_prior_destroy": (_I, [_P]),
    "jk_prior_load_layer": (_I, [_P, _I, C.POINTER(LayerWeights), _P]),
    "jk_prior_set_embeddings": (_I, [_P, _P, _P, _P, _P]),
    "jk_prior_reset": (_I, [_P, _I, _P]),
    "jk_prior_set_encoder_kv": (_I, [_P, _P, _I, _P]),
    "jk_prior_step": (_I, [_P, C.POINTER(StepArgs), _P]),
    "jk_prior_prefill_capacity": (_I, [_P, C.POINTER(C.c_int)]),
    "jk_prior_config_prefill_capacity": (_I, [C.POINTER(PriorConfig), C.POINTER(C.c_int)]),
    "jk_prior_prefill": (_I, [_P, C.POINTER(PrefillArgs), _P]),
    "jk_pool_rows_f32": (_I, [_P, _I, _I, _I, _I, _I, _P, _L, _P, _P]),
    "jk_prior_position": (_I, [_P, C.POINTER(C.c_int)]),
    "jk_prior_has_logits_gemm": (_I, [_P, C.POINTER(C.c_int)]),
    "jk_prior_select_plan": (_I, [C.POINTER(PriorConfig), C.POINTER(C.c_int32), _I, C.POINTER(SelectPlanInfo)]),
    "jk_prior_select": (_I, [_P, C.POINTER(C.c_int32), _I, _P, C.c_size_t, _P]),
    "jk_prior_debug_buffer": (_I, [_P, _I, C.POINTER(_P), C.POINTER(C.c_size_t)]),
    "jk_prefill_attention_f16": (_I, [C.POINTER(PrefillAttnArgs), C.POINTER(PrefillAttnRoute), _P]),
    "jk_conv1d_prefill_f16": (_I, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "jk_prefill_gemm_f16": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "jk_sample_categorical": (_I, [_P, _L, _I, _I, _F, C.c_uint64, _I, _P, _L, _P]),
    "jk_sample_categorical_scored": (_I, [_P, _L, _P, _L, _I, _I, _F, C.c_uint64, _I, _P, _L, _P, _L, _P]),
    "jk_xout_split_bytes": (_I, [_I, _I, C.POINTER(C.c_size_t)]),
    "jk_pack_xout_split": (_I, [_P, _P, _I, _I, _P]),
    "jk_xout_logprob_workspace_bytes": (_I, [_I, _I, _I, C.POINTER(C.c_size_t)]),
    "jk_xout_logprob": (_I, [_P, _I, _I, _P, _I, _P, _P, _P, _P, C.c_size_t, _P]),
    "jk_xout_stats_workspace_bytes": (_I, [_I, _I, _I, _I, C.POINTER(C.c_size_t)]),
    "jk_xout_stats": (_I, [_P, _I, _I, _P, _I, _P, _I, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "jk_filter_logits": (_I, [_P, _L, _I, _I, _F, _I, _F, _P, _L, _P]),
    "jk_sample_guided": (_I, [_P, _L, _P, _L, _I, _I, _F, _F, _I, _F, C.c_uint64, _I, _P, _L, _P, _L, _P, _P, _L, _P]),
    "jk_vq_argmin": (_I, [_P, _P, _P, _P, _L, _I, _I, _P]),
    "jk_vq_gather": (_I, [_P, _P, _P, _L, _I, _I, _P]),
    "jk_conv1d_cl": (_I, [C.POINTER(ConvArgs), _P]),
    "jk_conv_weight_split_bytes": (_I, [_I, _I, _I, C.POINTER(C.c_size_t)]),
    "jk_pack_conv_weight_split": (_I, [_P, _P, _I, _I, _I, _P]),
    "jk_conv1d_tc_wide": (_I, [C.POINTER(ConvArgs), _P, _P]),
    "jk_stft_mag_diff": (_I, [_P, _P, _P, _P, _P, _I, _L, _I, _I, _I, _P, C.c_size_t, _P]),
    "jk_stft_workspace_bytes": (C.c_size_t, [_I, _L, _I, _I]),
    "jk_resblock_cl": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _L, _I, _I, _I, _F, _P]),
    "jk_resblock_tc": (_I, [_P, _P, _P, _P, _P, _P, _I, _L, _I, _I, _F, _P]),
    "jk_pack_conv_weight": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "jk_layernorm_f32": (_I, [_P, _P, _P, _P, _L, _I, _F, _P]),
    "jk_embedding_f32": (_I, [_P, _P, _P, _P, _L, _I, _I, _P]),
    "jk_f32_workspace_floats": (_I, [C.POINTER(F32Args), C.POINTER(C.c_size_t)]),
    "jk_f32_forward": (_I, [C.POINTER(F32Args), C.POINTER(F32Layer), _P]),
    "jk_f32_embed": (_I, [_P, _P, _L, _P, _P, _L, _P, _P, _P, _I, _I, _I, _I, _P]),
    "jk_f32_linear": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "jk_f32_backward_workspace_floats": (_I, [C.POINTER(F32Args), C.POINTER(C.c_size_t)]),
    "jk_f32_backward": (_I, [C.POINTER(F32Args), C.POINTER(F32Layer), C.POINTER(F32GradLayer), C.POINTER(_P), _P, _P, _P]),
    "jk_f32_linear_wgrad": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "jk_f32_embed_backward": (_I, [_P, _P, _L, _I, _I, _I, _I, _P, _P, _P, _P, _I, _P]),
    "jk_f32_xent_backward": (_I, [_P, _P, _P, _P, _I, _I, _P]),
}

_lib = None


def lib():
    """The loaded shared library (loads it on first use; no alternative implementation exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing - build it with `python -m jukebox_b200.build` "
                "(jukebox_b200 has no CPU or pure-PyTorch path)")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


CALLS = 0      # C-ABI calls that enqueue GPU work (bench.py reports it as its launch evidence)


def check(rc):
    global CALLS
    CALLS += 1
    if rc != 0:
        raise RuntimeError("libjkb200: " + lib().jk_last_error().decode())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device pointer of a CUDA tensor (None -> NULL).  Non-CUDA tensors are an error: there is
    no host path."""
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise RuntimeError("jukebox_b200 kernels need CUDA tensors (no CPU fallback); got " + str(t.device))
    if not t.is_contiguous():
        raise RuntimeError("tensor must be contiguous")
    return C.c_void_p(t.data_ptr())


def sm_count():
    out = C.c_int(0)
    check(lib().jk_device_sm_count(C.byref(out)))
    return out.value
