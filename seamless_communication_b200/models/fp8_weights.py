"""FP8 decoder weights: the definition of the weight-only E4M3 mode of the text and unit searches (DESIGN.md section 16).

Each quantized weight W (one row per output feature: a projection row or a vocabulary row) is stored as e4m3fn bytes q
and one fp32 scale s per row:
  * s = 2^ceil(log2(amax / 448)) for the row's largest magnitude amax, clamped to [2^-15, 2^7]; an all-zero row has s = 1;
  * q = e4m3fn(W / s), rounded to nearest even; |W / s| <= 448, so it never saturates.
Because s is a power of two, W' = q * s is exactly an fp16 value.  The FP8 engine computes exactly the fp16 model with W
replaced by W' (`dequantize_decoder_weights`): nothing is approximate beyond the rounding of the weights themselves.
(One limit, DESIGN.md section 16: in rows far below the scale's clamp floor, whose W' are fp16 subnormals around 2^-24,
products near 2^-34 can differ in the last bits.)

Quantized, per decoder layer: the self-attention q / k / v / output projections, the cross-attention q and output
projections, FFN inner and output; and the tied embedding / final projection.  Not quantized: the cross-attention K|V
projections (computed once per utterance), biases and LayerNorms."""
from __future__ import annotations

from typing import Dict, List

import torch

E4M3_MAX = 448.0
SCALE_MIN_EXP, SCALE_MAX_EXP = -15, 7

_LAYER_WEIGHTS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.output_proj",
                  "encoder_decoder_attn.q_proj", "encoder_decoder_attn.output_proj", "ffn.inner_proj", "ffn.output_proj")


def quantize_rows(w: torch.Tensor):
    """(q float8_e4m3fn (n, k), s float32 (n,)) of a 2-D weight, one power-of-two scale per row.  ValueError for a
    non-finite weight or a row whose largest magnitude exceeds 448 * 2^7."""
    if w.dim() != 2:
        raise ValueError(f"expected a 2-D weight, got shape {tuple(w.shape)}")
    x = w.float()
    if not bool(torch.isfinite(x).all()):
        raise ValueError("cannot quantize a non-finite weight to e4m3")
    amax = x.abs().amax(dim=1)
    if bool((amax > E4M3_MAX * 2.0 ** SCALE_MAX_EXP).any()):
        raise ValueError(f"a weight row's magnitude exceeds {E4M3_MAX} * 2^{SCALE_MAX_EXP}, the largest e4m3 range of a scale")
    # smallest e with amax <= 448 * 2^e, exactly: amax = m * 2^E (m in [0.5, 1)), 448 = 0.875 * 2^9
    m, E = torch.frexp(amax)
    e = torch.where(m <= 0.875, E - 9, E - 8).clamp(SCALE_MIN_EXP, SCALE_MAX_EXP)
    e = torch.where(amax == 0, torch.zeros_like(e), e)
    s = torch.ldexp(torch.ones_like(amax), e)
    q = (x / s[:, None]).to(torch.float8_e4m3fn)  # exact division by a power of two, then round to nearest even
    return q, s


def dequantize_rows(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """W' = q * s in fp16 (exact)."""
    return (q.float() * s.float()[:, None]).half()


def decoder_weight_names(state_dict: Dict[str, torch.Tensor], cfg) -> List[str]:
    """State-dict names of the weights FP8 mode quantizes: the text decoder's (and, for an autoregressive T2U, the
    unit decoder's) six products per layer and the tied embedding / final projection, where present."""
    names: List[str] = []
    decoders = [("text_decoder.layers", cfg.dec_layers, ("text_decoder_frontend.embed.weight", "final_proj.weight"))]
    if cfg.encoder_variant == "v1":  # the AR T2U's unit decoder (the NAR T2U of v2 is out of scope)
        decoders.append(("t2u_model.decoder.layers", cfg.t2u_dec_layers,
                         ("t2u_model.decoder_frontend.embed.weight", "t2u_model.final_proj.weight")))
    for prefix, layers, tied in decoders:
        for i in range(layers):
            for p in _LAYER_WEIGHTS:
                k = f"{prefix}.{i}.{p}.weight"
                if k in state_dict:
                    names.append(k)
        names += [k for k in tied if k in state_dict]
    return names


def dequantize_decoder_weights(state_dict: Dict[str, torch.Tensor], cfg) -> Dict[str, torch.Tensor]:
    """The fp16 state dict of the FP8 model: every quantized weight (`decoder_weight_names`) replaced by W' = q * s,
    everything else as given.  An fp16 model built from it computes what the FP8 model computes, bit for bit."""
    out = dict(state_dict)
    for k in decoder_weight_names(state_dict, cfg):
        out[k] = dequantize_rows(*quantize_rows(state_dict[k]))
    return out
