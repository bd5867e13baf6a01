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
        ("fin_anc", c_p), ("n_active", c_p), ("len_budget", c_p), ("fin_scores", c_p),
    ]


# name -> argtypes (restype is int unless listed in _RESTYPES); must list every symbol include/seamless_b200.h declares
PROTOTYPES = {
    "sb_last_error": [],
    "sb_version": [],
    "sb_launch_count": [],
    "sb_pdl_enabled": [],
    "sb_gemm": [C.POINTER(GemmDesc), c_p],
    "sb_gemm_ref": [C.POINTER(GemmDesc), c_p],
    "sb_gemm_splitk": [C.POINTER(GemmDesc), i32, c_p, i64, c_p],
    "sb_gemm_decode_supported": [c_p, i32],
    "sb_gemm_decode": [c_p, i32, c_p, i64, c_p],
    "sb_gemm_decode_e4m3": [c_p, c_p, i32, c_p, i64, c_p],
    "sb_vocab_proj_e4m3": [C.POINTER(GemmDesc), c_p, c_p],
    "sb_splitk_reduce_ln": [c_p, i32, i32, i64, i32, c_p, c_p, c_p, c_p, c_p, c_p],
    "sb_fbank": [c_p, i64, c_p, i32, c_p, i32, c_p, c_p, i32, c_p],
    "sb_layernorm": [c_p, c_p, c_p, c_p, c_p, c_p, i32, i32, i32, i32, i32, i32, i32, c_p, i32, c_p],
    "sb_attention": [c_p, i64, c_p, i64, c_p, i64, c_p, i64, i32, i32, i32, i32, i32, i32, i32, i32, c_p, i32, c_p, i32,
                     i32, c_p],
    "sb_attention_relpos": [c_p, i64, c_p, i64, c_p, i64, c_p, i64, i32, i32, i32, i32, i32, i32, i32, c_p, c_p, i64, c_p,
                            c_p, c_p],
    "sb_w2v2_front": [c_p, i64, c_p, i32, c_p, c_p, c_p, c_p, c_p, i32, c_p, c_p],
    "sb_layernorm_gelu": [c_p, c_p, c_p, c_p, i32, i32, i32, i32, i32, i32, i32, c_p, i32, c_p],
    "sb_attention_hd80": [c_p, i64, c_p, i64, c_p, i64, c_p, i64, i32, i32, i32, i32, i32, i32, i32, i32, c_p, c_p],
    "sb_nearest_centroid": [c_p, i64, i32, i32, c_p, c_p, i32, i32, c_p, c_p, c_p, c_p],
    "sb_align_lprob": [c_p, i64, i32, i32, c_p, c_p, i64, i32, i32, c_p, i32, i32, i32, i32, f32, c_p, i64, c_p],
    "sb_monotonic_align": [c_p, i64, i32, i32, i32, c_p, c_p, c_p, c_p, c_p, c_p],
    "sb_dwconv_ln_silu": [c_p, c_p, c_p, c_p, c_p, i32, i32, i32, i32, c_p],
    "sb_dwconv_bias_silu": [c_p, c_p, c_p, c_p, i32, i32, i32, i32, c_p],
    "sb_embed_step": [c_p, i32, c_p, c_p, c_p, f32, c_p, i32, i32, c_p],
    "sb_step_advance": [c_p, c_p],
    "sb_store_step": [c_p, c_p, c_p, i64, c_p],
    "sb_embed_seq": [c_p, i32, i32, c_p, c_p, f32, c_p, i32, i32, c_p],
    "sb_decode_self_attn": [c_p, c_p, i32, i64, c_p, c_p, c_p, c_p, i32, c_p, i32, c_p, i32, i32, c_p],
    "sb_decode_cross_attn": [c_p, c_p, i32, i64, c_p, c_p, c_p, i64, c_p, i32, c_p, i32, i32, i32, c_p],
    "sb_decode_cross_attn_weights": [c_p, i32, i64, c_p, c_p, i64, c_p, i32, c_p, c_p, i32, i32, i32, c_p],
    "sb_logits_topk": [c_p, i64, i32, i32, i32, i32, i32, f32, i32, c_p, c_p, c_p, c_p],
    "sb_logits_topk_tiles": [c_p, i64, c_p, i32, i32, i32, i32, i32, f32, i32, c_p, c_p, c_p, c_p],
    "sb_beam_step": [C.POINTER(BeamDesc), c_p],
    "sb_token_timestamps": [c_p, i32, i32, c_p, i32, c_p, c_p, i32, i32, i32, c_p, i64, c_p, i32, c_p],
    "sb_ban_step": [c_p, i32, c_p, i32, c_p, i32, i32, c_p, c_p, c_p],
    "sb_ngram_ban_step": [c_p, i32, c_p, i32, i32, i32, c_p, c_p, c_p],
    "sb_logits_topk_ban": [c_p, i64, i32, i32, i32, i32, i32, f32, i32, c_p, c_p, c_p, c_p, c_p, i32, c_p],
    "sb_logits_topk_tiles_ban": [c_p, i64, c_p, i32, i32, i32, i32, i32, f32, i32, c_p, c_p, c_p, c_p, c_p, i32, c_p],
    "sb_text_to_chars": [c_p, i32, i32, c_p, c_p, c_p, i32, i32, i32, i32, c_p, c_p, i32, c_p, c_p],
    "sb_upsample_add": [c_p, i32, i32, i32, c_p, c_p, i32, i32, i32, i32, i32, c_p, c_p, c_p, c_p, i32, f32, c_p, c_p],
    "sb_durations": [c_p, i32, i32, c_p, f32, i32, c_p, i32, i32, f32, c_p, c_p],
    "sb_unit_argmax": [c_p, i64, i32, i32, i32, i32, i32, c_p, i32, i32, c_p, c_p],
    "sb_hifigan_resblock": [c_p, c_p],
    "sb_vocoder_embed": [c_p, i32, i32, c_p, i32, c_p, i32, c_p, c_p, i32, c_p, c_p, i32, i32, c_p],
    "sb_conv_post_tanh": [c_p, i32, i32, i32, c_p, i32, i32, c_p, f32, i32, c_p, i64, c_p],
    "sb_avgpool_time": [c_p, c_p, i32, i32, i32, i32, c_p],
    "sb_pchoose": [c_p, c_p, c_p, i32, i32, i32, f32, f32, c_p],
    "sb_pchoose_ragged": [c_p, i32, c_p, i32, c_p, c_p, c_p, i32, i32, f32, f32, c_p],
    "sb_policy_decide": [c_p, i64, i32, c_p, c_p, i32, i32, i32, c_p, c_p],
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
