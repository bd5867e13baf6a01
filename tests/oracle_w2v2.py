"""fp32 torch restatement of the reference's UnitExtractor.predict (models/unit_extractor/unit_extractor.py:62-98) with
the xlsr2_1b_v2 encoder and KmeansModel.forward (kmeans.py:14-30), for the unit-extractor tests.

Items marked [fs2-recall] live in fairseq2, which is not in the reference tree; they are written here as recalled:
  * the feature extractor's layer order in layer_norm mode: Conv1d(bias) -> LayerNorm over channels -> GELU, per layer;
  * the frontend: post_extract_layer_norm -> model_dim_proj -> padded frames zeroed -> x + GELU(pos_conv(x)), pos_conv a
    weight-normed (dim 2) grouped Conv1d with padding K/2 whose last output frame is dropped; no frontend LayerNorm under
    norm_order PRE;
  * the encoder layer: pre-LN self-attention (scale head_dim^-0.5, key padding mask) and pre-LN FFN with GELU; the
    layer-output hook returns layer out_layer_idx's output before encoder.layer_norm.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def collate(wave: Tensor) -> Tuple[Tensor, int]:
    """Collater(pad_value=1, pad_to_multiple=2) of one 1-D waveform: (Lp,) samples and the unpadded length L."""
    L = wave.shape[0]
    if L % 2:
        wave = torch.cat([wave, torch.ones(1, dtype=wave.dtype)])
    return wave, L


def conv_frames(n: int, descs) -> int:
    for _, k, s in descs:
        n = (n - k) // s + 1 if n >= k else 0
    return n


def feature_extractor(x: Tensor, sd: Dict[str, Tensor], descs) -> Tensor:
    """x (Lp,) normalised samples -> (T, 512) [fs2-recall: conv -> LayerNorm -> GELU per layer]."""
    h = x.reshape(1, 1, -1)
    for i, (c, k, s) in enumerate(descs):
        p = f"encoder_frontend.feature_extractor.layers.{i}"
        h = F.conv1d(h, sd[p + ".conv.weight"], sd[p + ".conv.bias"], stride=s)
        h = F.layer_norm(h.transpose(1, 2), (c,), sd[p + ".layer_norm.weight"], sd[p + ".layer_norm.bias"], 1e-5).transpose(1, 2)
        h = F.gelu(h)
    return h[0].transpose(0, 1)


def pos_conv_weight(sd: Dict[str, Tensor]) -> Tensor:
    """weight_norm(dim=2): w[:, :, k] = g[k] v[:, :, k] / ||v[:, :, k]||"""
    p = "encoder_frontend.pos_encoder.conv"
    v, g = sd[p + ".weight_v"], sd[p + ".weight_g"].reshape(-1)
    return v * (g / v.pow(2).sum((0, 1)).sqrt())[None, None, :]


def frontend(feats: Tensor, mask_len: int, sd: Dict[str, Tensor], cfg) -> Tensor:
    """(T, 512) -> (T, M) [fs2-recall]"""
    x = F.layer_norm(feats, (feats.shape[1],), sd["encoder_frontend.post_extract_layer_norm.weight"],
                     sd["encoder_frontend.post_extract_layer_norm.bias"], 1e-5)
    x = F.linear(x, sd["encoder_frontend.model_dim_proj.weight"], sd["encoder_frontend.model_dim_proj.bias"])
    x = x.clone()
    x[mask_len:] = 0
    K = cfg.pos_conv_kernel_size
    y = F.conv1d(x.t()[None], pos_conv_weight(sd), sd["encoder_frontend.pos_encoder.conv.bias"], padding=K // 2,
                 groups=cfg.num_pos_conv_groups)
    if K % 2 == 0:
        y = y[:, :, :-1]
    return x + F.gelu(y[0].t())


def encoder_layer(x: Tensor, mask_len: int, sd: Dict[str, Tensor], p: str, H: int,
                  act: Callable[[Tensor], Tensor] = F.gelu) -> Tensor:
    """One pre-LN Transformer encoder layer [fs2-recall] on (T, M)."""
    T, M = x.shape
    d = M // H
    h = F.layer_norm(x, (M,), sd[p + ".self_attn_layer_norm.weight"], sd[p + ".self_attn_layer_norm.bias"], 1e-5)
    q, k, v = (F.linear(h, sd[f"{p}.self_attn.{n}_proj.weight"], sd[f"{p}.self_attn.{n}_proj.bias"]).reshape(T, H, d).transpose(0, 1)
               for n in "qkv")
    s = q @ k.transpose(1, 2) * d ** -0.5
    s[:, :, mask_len:] = float("-inf")
    a = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(T, M)
    x = x + F.linear(a, sd[p + ".self_attn.output_proj.weight"], sd[p + ".self_attn.output_proj.bias"])
    h = F.layer_norm(x, (M,), sd[p + ".ffn_layer_norm.weight"], sd[p + ".ffn_layer_norm.bias"], 1e-5)
    t = act(F.linear(h, sd[p + ".ffn.inner_proj.weight"], sd[p + ".ffn.inner_proj.bias"]))
    return x + F.linear(t, sd[p + ".ffn.output_proj.weight"], sd[p + ".ffn.output_proj.bias"])


def features(wave: Tensor, sd: Dict[str, Tensor], cfg, out_layer_idx: int) -> Tuple[Tensor, int]:
    """Steps 1-5: the output of encoder layer out_layer_idx, (T, M) for every frame of the collated sequence, and the
    padding-mask frame count."""
    descs = cfg.feature_extractor_layer_descs
    x, L = collate(wave.float())
    x = F.layer_norm(x[None], x[None].shape, eps=1e-5)[0]
    mask_len = conv_frames(L, descs)
    h = frontend(feature_extractor(x, sd, descs), mask_len, sd, cfg)
    for i in range(out_layer_idx + 1):
        h = encoder_layer(h, mask_len, sd, f"encoder.layers.{i}", cfg.num_encoder_attn_heads)
    return h, mask_len


def kmeans(x: Tensor, centroids: Tensor) -> Tensor:
    """KmeansModel.forward: argmin(|x|^2 - 2 x.C^T + |c|^2), ties to the lowest index; centroids (K, D)."""
    c = centroids.t()
    dist = x.pow(2).sum(1, keepdim=True) - 2 * x @ c + c.pow(2).sum(0, keepdim=True)
    return dist.argmin(dim=-1)


def predict(wave: Tensor, sd: Dict[str, Tensor], cfg, centroids: Tensor, out_layer_idx: int) -> Tuple[Tensor, Tensor]:
    h, _ = features(wave, sd, cfg, out_layer_idx)
    return kmeans(h, centroids), h


def distance_gaps(x: Tensor, centroids: Tensor, a: Tensor, b: Tensor) -> Tensor:
    """fp64 |x - c_a|^2 - |x - c_b|^2 per row (the near-tie audit)."""
    x, c = x.double(), centroids.double()
    return (x - c[a]).pow(2).sum(1) - (x - c[b]).pow(2).sum(1)
