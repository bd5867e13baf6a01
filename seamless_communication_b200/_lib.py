"""ctypes binding of the C-ABI library (include/seamless_b200.h).

The product path has no CPU fallback: if `libseamless_b200.so` is missing, or no CUDA device is present when a
kernel is requested, a RuntimeError is raised (build with `python -c "import __graft_entry__ as g; g.build()"`).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libseamless_b200.so")

c_p = C.c_void_p
i32, i64, f32 = C.c_int32, C.c_int64, C.c_float


class GemmDesc(C.Structure):
    _fields_ = [
        ("a", c_p), ("a_rows", i64), ("a_ld", i64), ("c_in", i32), ("taps", i32), ("dil", i32), ("a_row0", i32),
        ("w", c_p), ("n", i32), ("m", i32), ("bias", c_p), ("act", i32), ("act_slope", f32), ("glu", i32),
        ("alpha", f32), ("gamma", f32), ("res1", c_p), ("res1_ld", i64), ("res2", c_p), ("res2_ld", i64),
        ("out", c_p), ("out_ld", i64), ("out_f32", i32), ("out2", c_p), ("out2_ld", i64), ("out2_slope", f32),
        ("out_row0", i64), ("seq_rows", i32), ("seq_halo", i32), ("seq_len", i32), ("seq_lens", c_p),
        ("prefetch", c_p), ("prefetch_bytes", i64), ("tile_stats", c_p),
    ]


class ResblockDesc(C.Structure):
    _fields_ = [
        ("x", c_p), ("res2", c_p), ("out", c_p), ("out2", c_p),
        ("w1", c_p * 3), ("b1", c_p * 3), ("w2", c_p * 3), ("b2", c_p * 3),
        ("dilation", i32 * 3), ("channels", i32), ("kernel_size", i32),
        ("batch", i32), ("T", i32), ("rows_per_seq", i32), ("halo", i32),
        ("slope", f32), ("gamma", f32), ("out2_slope", f32), ("lens", c_p),
    ]


class BeamDesc(C.Structure):
    _fields_ = [
        ("batch", i32), ("beam", i32), ("max_len", i32), ("vocab", i32), ("K", i32),
        ("step_ptr", c_p), ("prefix_len", i32), ("eos_idx", i32), ("min_len", i32), ("len_penalty", f32),
        ("cand_val", c_p), ("cand_idx", c_p), ("eos_lprob", c_p),
        ("seqs", c_p), ("scores", c_p), ("anc", c_p),
        ("fin_count", c_p), ("fin_score", c_p), ("fin_len", c_p), ("fin_seqs", c_p), ("active", c_p),
        ("fin_anc", c_p), ("n_active", c_p), ("len_budget", c_p),
    ]


class DecoderLayerDesc(C.Structure):
    _fields_ = [(n, c_p) for n in (
        "qkv_b", "out_b", "cq_b", "co_b", "ffn1_b", "ffn2_b",
        "ca_ln_w", "ca_ln_b", "ffn_ln_w", "ffn_ln_b", "next_ln_w", "next_ln_b", "k_cache", "v_cache", "cross_k", "cross_v")
    ]


class DecoderPlanDesc(C.Structure):
    _fields_ = [
        ("layers", i32), ("dim", i32), ("ffn_dim", i32), ("heads", i32), ("rows", i32), ("beam", i32), ("groups", i32),
        ("max_len", i32), ("s_enc", i32),
        ("layer", C.POINTER(DecoderLayerDesc)), ("w_dim_stack", c_p), ("w_ffn_stack", c_p), ("ln0_w", c_p), ("ln0_b", c_p), ("embed", c_p), ("pos", c_p),
        ("embed_scale", f32), ("seqs", c_p), ("seqs_ld", i32), ("anc", c_p), ("anc_ld", i32), ("step_ptr", c_p),
        ("enc_lens", c_p), ("x", c_p), ("h", c_p), ("att", c_p), ("ffn_act", c_p),
        ("part_qkv", c_p), ("part_qkv_floats", i64), ("part", c_p), ("part_floats", i64), ("hist", c_p),
        ("counters", c_p), ("counters_len", i64), ("timeline", c_p),
    ]


class DecoderPlanInfo(C.Structure):
    _fields_ = [
        ("part_qkv_floats", i64), ("part_floats", i64), ("counters_len", i64),
        ("groups", i32), ("rows_per_group", i32), ("npad", i32), ("ctas_per_group", i32), ("stages", i32),
        ("smem_bytes", i32), ("n_phases", i32), ("splits", i32 * 6),
    ]


class DecoderLaunch(C.Structure):
    _fields_ = [("counters", c_p), ("counters_len", i64), ("grid", i32), ("block", i32),
                ("smem_bytes", i32), ("cooperative", i32), ("npad", i32), ("reserved", i32), ("params", C.c_uint64 * 768)]


# name -> argtypes (restype is int unless listed in _RESTYPES); must list every symbol include/seamless_b200.h declares
PROTOTYPES = {
    "sb_last_error": [],
    "sb_version": [],
    "sb_launch_count": [],
    "sb_gemm": [C.POINTER(GemmDesc), c_p],
    "sb_gemm_ref": [C.POINTER(GemmDesc), c_p],
    "sb_gemm_splitk": [C.POINTER(GemmDesc), i32, c_p, i64, c_p],
    "sb_gemm_decode_supported": [c_p, i32],
    "sb_gemm_decode": [c_p, i32, c_p, i64, c_p],
    "sb_splitk_reduce_ln": [c_p, i32, i32, i64, i32, c_p, c_p, c_p, c_p, c_p, c_p],
    "sb_fbank": [c_p, i64, c_p, i32, c_p, i32, c_p, c_p, i32, c_p],
    "sb_layernorm": [c_p, c_p, c_p, c_p, c_p, c_p, i32, i32, i32, i32, i32, i32, i32, c_p, i32, c_p],
    "sb_attention": [c_p, i64, c_p, i64, c_p, i64, c_p, i64, i32, i32, i32, i32, i32, i32, i32, i32, c_p, i32, c_p, i32,
                     i32, c_p],
    "sb_attention_relpos": [c_p, i64, c_p, i64, c_p, i64, c_p, i64, i32, i32, i32, i32, i32, i32, i32, c_p, c_p, i64, c_p,
                            c_p, c_p],
    "sb_dwconv_ln_silu": [c_p, c_p, c_p, c_p, c_p, i32, i32, i32, i32, c_p],
    "sb_dwconv_bias_silu": [c_p, c_p, c_p, c_p, i32, i32, i32, i32, c_p],
    "sb_embed_step": [c_p, i32, c_p, c_p, c_p, f32, c_p, i32, i32, c_p],
    "sb_step_advance": [c_p, c_p],
    "sb_store_step": [c_p, c_p, c_p, i64, c_p],
    "sb_embed_seq": [c_p, i32, i32, c_p, c_p, f32, c_p, i32, i32, c_p],
    "sb_decode_self_attn": [c_p, c_p, i32, i64, c_p, c_p, c_p, c_p, i32, c_p, i32, c_p, i32, i32, c_p],
    "sb_decode_cross_attn": [c_p, c_p, i32, i64, c_p, c_p, c_p, i64, c_p, i32, c_p, i32, i32, i32, c_p],
    "sb_logits_topk": [c_p, i64, i32, i32, i32, i32, i32, f32, i32, c_p, c_p, c_p, c_p],
    "sb_logits_topk_tiles": [c_p, i64, c_p, i32, i32, i32, i32, i32, f32, i32, c_p, c_p, c_p, c_p],
    "sb_beam_step": [C.POINTER(BeamDesc), c_p],
    "sb_kv_heads_major": [c_p, i64, i32, i32, i32, c_p, c_p, c_p],
    "sb_decoder_plan_query": [i32, i32, i32, i32, i32, i32, C.POINTER(DecoderPlanInfo)],
    "sb_decoder_plan_init": [C.POINTER(DecoderPlanDesc), C.POINTER(DecoderLaunch)],
    "sb_decoder_step": [C.POINTER(DecoderLaunch), c_p],
    "sb_text_to_chars": [c_p, i32, i32, c_p, c_p, c_p, i32, i32, i32, i32, c_p, c_p, i32, c_p, c_p],
    "sb_upsample_add": [c_p, i32, i32, i32, c_p, c_p, i32, i32, i32, i32, i32, c_p, c_p, c_p, c_p, i32, f32, c_p, c_p],
    "sb_durations": [c_p, i32, i32, c_p, f32, i32, c_p, i32, i32, f32, c_p, c_p],
    "sb_unit_argmax": [c_p, i64, i32, i32, i32, i32, i32, c_p, i32, i32, c_p, c_p],
    "sb_hifigan_resblock": [c_p, c_p],
    "sb_vocoder_embed": [c_p, i32, i32, c_p, i32, c_p, i32, c_p, c_p, i32, c_p, c_p, i32, i32, c_p],
    "sb_conv_post_tanh": [c_p, i32, i32, i32, c_p, i32, i32, c_p, f32, i32, c_p, i64, c_p],
    "sb_avgpool_time": [c_p, c_p, i32, i32, i32, i32, c_p],
    "sb_pchoose": [c_p, c_p, c_p, i32, i32, i32, f32, f32, c_p],
    "sb_cast_f32_to_f16": [c_p, c_p, i64, c_p],
    "sb_fill_zero": [c_p, i64, c_p],
}
_RESTYPES = {"sb_last_error": C.c_char_p, "sb_launch_count": i64}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Loads the shared library and binds every prototype.  Works without a GPU (symbol check only)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: the CUDA extension is not built (run __graft_entry__.build()); "
                "seamless_communication_b200 has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, args in PROTOTYPES.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = _RESTYPES.get(name, C.c_int)
        _lib = lib
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().sb_last_error()
        raise RuntimeError(f"{what or 'seamless_b200'} failed (code {rc}): {msg.decode() if msg else ''}")


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise RuntimeError("seamless_communication_b200 needs a CUDA device (sm_90a); there is no CPU fallback.")
    return load()
