"""CPU oracle of the w2v-BERT v1 speech encoder (seamlessM4T_large), test infrastructure like oracle/unity_oracle.py.

`UnityOracle` already restates the v1 Conformer block behind variant="v1" (pinned against the reference's compiled C++,
tests/golden/conformer_v1_ref.npz), but its `mha_relpos_v1` runs one unpadded sequence only.  This subclass adds what a
ragged batch needs and leaves the pinned code untouched:
  * `mha_relpos`: RelativePositionSDPA over a padded batch with the key padding mask, through the closed form
    R[S-1+j-i] of the relative shift (`shift_bd` below is the oracle's pad/reshape/slice, fairseq2.cpp:661-675);
  * `encode_speech`: the v1 stack (frontend -> v1 Conformer layers -> adaptor) with the recalled position table
    (`relpos_table`) or, when the state dict carries one, `speech_encoder.pos_enc`.

What is pinned and what is recalled (DESIGN.md §8):
  * pinned by the C++ mirror: the block order, conv module order (GLU, symmetric depthwise padding, eval BatchNorm,
    SiLU), the u / v biases and r_proj of RelativePositionSDPA, the relative shift and the table slice
    [n_ctx-S, n_ctx+S-1) with n_ctx = 4096 (fairseq2.cpp:605-756);
  * [fs2-recall]: the table formula (RelativePositionalEncoding), the key padding mask inside RelativePositionSDPA (the
    mirror runs unpadded sequences), the zeroing of padded frames before pointwise_conv1 in v1, and the architecture
    hyper-parameters of seamlessM4T_large (builder.py:109-134, the 600m / dense_1b dims of base_v2).
"""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.unity_oracle import UnityOracle, key_mask  # noqa: E402

N_CTX = 4096


def relpos_table(n_ctx: int, dim: int) -> torch.Tensor:
    """[fs2-recall] RelativePositionalEncoding: row r holds step n_ctx-1-r (rows 0..n_ctx-1: n_ctx-1 .. 0, then -1 ..
    -(n_ctx-1)); column 2i = sin(step * exp(-2i ln(1e4)/dim)), column 2i+1 = cos of the same angle."""
    table = torch.zeros(2 * n_ctx - 1, dim)
    steps = torch.arange(n_ctx - 1, -n_ctx, -1, dtype=torch.float32)[:, None]
    freq = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))[None, :]
    table[:, 0::2] = torch.sin(steps * freq)
    table[:, 1::2] = torch.cos(steps * freq)
    return table


def shift_bd(bd: torch.Tensor) -> torch.Tensor:
    """The relative shift of `UnityOracle.mha_relpos_v1` (fairseq2 _shift_bd, mirrored fairseq2.cpp:661-675):
    (..., S, 2S-1) -> (..., S, S)."""
    N, H, S, _ = bd.shape
    return F.pad(bd, (1, 0)).view(N, H, 2 * S, S)[:, :, 1:].reshape(N, H, S, 2 * S - 1)[..., :S]


def relpos_index(S: int) -> torch.Tensor:
    """Closed form of the shift: score (i, j) reads column S-1+j-i of the (S, 2S-1) positional scores."""
    return S - 1 + torch.arange(S)[None, :] - torch.arange(S)[:, None]


class UnityOracleV1(UnityOracle):
    def __init__(self, cfg, sd, tokenizers=None):
        super().__init__(cfg, sd, tokenizers)
        pe = sd.get("speech_encoder.pos_enc")
        self.pos_enc = pe if pe is not None else relpos_table(N_CTX, self.M)

    def mha_relpos(self, p, x, km=None):
        """RelativePositionSDPA over a padded batch: scores ((q+u).k_j + (q+v).R[S-1+j-i]) / 8, keys j >= len masked."""
        N, S, _ = x.shape
        H, K = self.H, self.M // self.H
        q = self.lin(x, p + ".q_proj").view(N, S, H, K).transpose(1, 2)
        k = self.lin(x, p + ".k_proj").view(N, S, H, K).transpose(1, 2)
        v = self.lin(x, p + ".v_proj").view(N, S, H, K).transpose(1, 2)
        pe = self.pos_enc.to(x.device)
        r = F.linear(pe[N_CTX - S:N_CTX + S - 1], self.sd[p + ".sdpa.r_proj.weight"]).view(2 * S - 1, H, K).transpose(0, 1)
        u, vb = self.sd[p + ".sdpa.u_bias"].view(H, 1, K), self.sd[p + ".sdpa.v_bias"].view(H, 1, K)
        ac = torch.matmul(q + u, k.transpose(2, 3))
        bd = torch.matmul(q + vb, r.transpose(1, 2))                                   # (N,H,S,2S-1)
        bd = torch.gather(bd, 3, relpos_index(S).to(x.device).expand(N, H, S, S))
        w = (ac + bd) * (K ** -0.5)
        if km is not None:
            w = w.masked_fill(~km[:, None, None, :].to(x.device), float("-inf"))
        a = torch.softmax(w, dim=-1)
        return self.lin(torch.matmul(a, v).transpose(1, 2).reshape(N, S, self.M), p + ".output_proj")

    def conformer_layer_v1(self, x, i, km):
        """`UnityOracle.conformer_layer(variant="v1")` with the masked attention above."""
        p = f"speech_encoder.inner.layers.{i}"
        x = x + 0.5 * self.ffn(self.ln(x, p + ".ffn1_layer_norm"), p + ".ffn1", F.silu)
        x = x + self.mha_relpos(p + ".self_attn", self.ln(x, p + ".self_attn_layer_norm"), km)
        x = x + self.conformer_conv(self.ln(x, p + ".conv_layer_norm"), p + ".conv", km, "v1")
        x = x + 0.5 * self.ffn(self.ln(x, p + ".ffn2_layer_norm"), p + ".ffn2", F.silu)
        return self.ln(x, p + ".layer_norm")

    def encode_speech(self, fb, lens=None, return_inner=False):
        x, lens = self.speech_frontend(fb, lens)
        km = key_mask(lens.cpu() if lens is not None else None, x.shape[1])
        km = km.to(x.device) if km is not None else None
        if x.shape[1] > N_CTX:
            raise ValueError(f"sequence length {x.shape[1]} exceeds {N_CTX}")
        for i in range(self.c["enc_layers"]):
            x = self.conformer_layer_v1(x, i, km)
        inner = x
        x, lens = self.encoder_adaptor(x, lens)
        return (x, lens, inner) if return_inner else (x, lens)

