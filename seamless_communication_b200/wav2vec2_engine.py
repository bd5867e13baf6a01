"""Host-side orchestration of the XLS-R unit extractor (DESIGN.md section 11) on the C-ABI kernels.

`Wav2Vec2Engine` packs a wav2vec2 encoder (fairseq2 names, models/checkpoint.py `convert_wav2vec2_checkpoint`) and a k-means
codebook once, and runs a batch of waveforms with per-row sample counts through
  sb_w2v2_front (statistics + conv 0 + LayerNorm + GELU) -> conv layers 1-6 on sb_gemm, each followed by
  sb_layernorm_gelu -> post-extract LayerNorm -> model_dim_proj (padded frames zeroed) -> positional conv (one sb_gemm per
  group, GELU and residual in the epilogue) -> encoder layers 0..out_layer_idx -> sb_nearest_centroid.

Frame layouts.  Conv layers 1-6 have stride 2: a (T, 512) activation viewed as (T/2, 1024) pair rows turns k2/s2 into one
tap over K = 1024 and k3/s2 into two taps (the second tap's upper 512 weight columns zero).  So every sequence owns a
block of Tp0 rows with Tp0 a multiple of 64, halved by each layer.  The positional conv runs on blocks with at least 64
zero rows after each sequence, which are the conv's zero padding for its own tail and its successor's head; the encoder
layers then run on a dense copy with one block of T rows per sequence (T = the batch's longest frame count).

Frame counts.  A row of L samples is collated to Lp = L + (L & 1) (an odd row gets a sample of value 1.0); its units cover
frames(Lp), while the padding mask (zeroed frames after the projection, the attention key mask) keeps frames(L), which
can be one fewer (unit_extractor.py:83-93 with Collater(pad_value=1, pad_to_multiple=2)).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib, ops
from .config import Wav2Vec2EncoderConfig
from .ops import ACT_GELU, F16, Seq

I32 = torch.int32
GEMM_MAX_ROW_TILES = 65535  # sb_gemm puts the 128-row tiles of M on gridDim.y
MIN_SAMPLES = 400  # fewer samples give no frame after the feature extractor


def conv_frames(n: int, descs: Sequence[Tuple[int, int, int]]) -> List[int]:
    """Frames after each feature-extractor layer for n input samples: floor((L - k) / s) + 1 per layer (0 when L < k)."""
    out = []
    for _, k, s in descs:
        n = (n - k) // s + 1 if n >= k else 0
        out.append(n)
    return out


class Wav2Vec2Engine:
    def __init__(self, cfg: Wav2Vec2EncoderConfig, state_dict: Dict[str, torch.Tensor], centroids: torch.Tensor, device="cuda"):
        _lib.require_cuda()
        descs = tuple(tuple(d) for d in cfg.feature_extractor_layer_descs)
        if cfg.head_dim != 80 or cfg.model_dim // cfg.num_pos_conv_groups != 80:
            raise ValueError("the unit extractor's kernels need head_dim 80 and 80 channels per positional-conv group")
        if descs[0] != (cfg.feature_dim, 10, 5) or cfg.feature_dim != 512 or \
                any(d not in ((512, 3, 2), (512, 2, 2)) for d in descs[1:]) or cfg.pos_conv_kernel_size % 2:
            raise ValueError("the feature extractor kernels need conv 0 = (512, 10, 5), then (512, 3, 2) / (512, 2, 2) layers, "
                             "and an even positional-conv kernel")
        if centroids.dim() != 2 or centroids.shape[1] != cfg.model_dim:
            raise ValueError(f"k-means centroids of shape {tuple(centroids.shape)} do not match model_dim {cfg.model_dim}")
        self.cfg, self.descs = cfg, descs
        self.device = torch.device(device)
        self.M, self.H = cfg.model_dim, cfg.num_encoder_attn_heads
        self._pack(state_dict, centroids)

    # ------------------------------------------------------------------------------------------ weight packing
    def _pack(self, sd, centroids):
        dev, cfg = self.device, self.cfg
        w: Dict[str, torch.Tensor] = {}

        def h(t):
            return t.to(dev, F16).contiguous()

        def f(t):
            return t.to(dev, torch.float32).contiguous()

        def lin(name):
            w[name + ".w"], w[name + ".b"] = h(sd[name + ".weight"]), f(sd[name + ".bias"])

        def ln(name):
            w[name + ".w"], w[name + ".b"] = f(sd[name + ".weight"]), f(sd[name + ".bias"])

        fe = "encoder_frontend.feature_extractor.layers"
        w["fe0.w"] = f(sd[f"{fe}.0.conv.weight"].reshape(512, 10))
        w["fe0.b"] = f(sd[f"{fe}.0.conv.bias"])
        ln(f"{fe}.0.layer_norm")
        for i, (c, k, _) in enumerate(self.descs[1:], 1):
            cw = sd[f"{fe}.{i}.conv.weight"]  # (512, 512, k): tap j of frame t reads input frame 2t + j
            pair0 = torch.cat([cw[:, :, 0], cw[:, :, 1]], 1)  # K index of pair row t: [x[2t] | x[2t+1]]
            if k == 3:
                pair1 = torch.cat([cw[:, :, 2], torch.zeros_like(cw[:, :, 2])], 1)  # pair row t+1: [x[2t+2] | unused]
                pair0 = torch.cat([pair0, pair1], 1)
            w[f"fe{i}.w"], w[f"fe{i}.b"] = h(pair0), f(sd[f"{fe}.{i}.conv.bias"])
            ln(f"{fe}.{i}.layer_norm")
        ln("encoder_frontend.post_extract_layer_norm")
        lin("encoder_frontend.model_dim_proj")
        # weight norm over dim 2 folded in fp64: w[:, :, k] = g[k] * v[:, :, k] / ||v[:, :, k]||, then one (80, K*80)
        # tap-major matrix per group
        p = "encoder_frontend.pos_encoder.conv"
        v, g = sd[p + ".weight_v"].double(), sd[p + ".weight_g"].double().reshape(-1)
        wn = v * (g / v.pow(2).sum((0, 1)).sqrt())[None, None, :]
        G, K = cfg.num_pos_conv_groups, cfg.pos_conv_kernel_size
        cg = self.M // G
        self.pos_w = [h(wn[i * cg:(i + 1) * cg].permute(0, 2, 1).reshape(cg, K * cg)) for i in range(G)]
        w["pos.b"] = f(sd[p + ".bias"])
        for i in range(cfg.num_encoder_layers):
            q = f"encoder.layers.{i}"
            ln(q + ".self_attn_layer_norm")
            w[q + ".qkv.w"] = h(torch.cat([sd[f"{q}.self_attn.{n}_proj.weight"] for n in "qkv"], 0))
            w[q + ".qkv.b"] = f(torch.cat([sd[f"{q}.self_attn.{n}_proj.bias"] for n in "qkv"], 0))
            lin(q + ".self_attn.output_proj")
            ln(q + ".ffn_layer_norm")
            lin(q + ".ffn.inner_proj")
            lin(q + ".ffn.output_proj")
        # KmeansModel: the CUDA path multiplies fp16 centroids, so |c|^2 is taken (in fp64) of exactly those values
        c16 = centroids.to(F16)
        w["km.c"] = c16.to(dev).contiguous()
        w["km.nhn"] = f(-0.5 * c16.double().pow(2).sum(1))
        self.w = w

    # ------------------------------------------------------------------------------------------ forward
    def frame_counts(self, num_samples: Sequence[int]) -> Tuple[List[List[int]], List[int]]:
        """Per row: frames after every conv layer of the collated Lp samples, and the padding-mask frame count of L."""
        per_layer = [conv_frames(n + (n & 1), self.descs) for n in num_samples]
        mask = [conv_frames(n, self.descs)[-1] for n in num_samples]
        return per_layer, mask

    def check_batch(self, num_samples: Sequence[int]) -> None:
        """ValueError for rows without a frame and for batches whose buffers exceed one kernel launch."""
        B = len(num_samples)
        if B == 0:
            raise ValueError("empty batch")
        if min(num_samples) < MIN_SAMPLES:
            raise ValueError(f"an input of {min(num_samples)} samples has no frame; the unit extractor needs at least {MIN_SAMPLES}")
        if B > 65535:
            raise ValueError(f"batch of {B} rows exceeds the kernels' limit of 65535 sequences per launch")
        per_layer = [conv_frames(n + (n & 1), self.descs) for n in num_samples]
        Tp0 = (max(pl[0] for pl in per_layer) + 63) // 64 * 64
        Te = (max(pl[-1] for pl in per_layer) + self.cfg.pos_conv_kernel_size // 2 + 7) // 8 * 8
        rows = B * max(Tp0 // 2, Te)  # the largest GEMM: conv 1 on pair rows, or the positional conv
        if (rows + 127) // 128 > GEMM_MAX_ROW_TILES:
            raise ValueError(f"batch needs {(rows + 127) // 128} row tiles in one sb_gemm launch; the limit is "
                             f"{GEMM_MAX_ROW_TILES} (65535 x 128 rows): split the batch")

    @torch.inference_mode()
    def forward(self, wave: torch.Tensor, num_samples: Sequence[int], out_layer_idx: int,
                marks: Optional[List[torch.cuda.Event]] = None) -> Tuple[Seq, List[int]]:
        """wave (B, T) fp32 on the device, row b valid up to num_samples[b] (nothing past it is read) -> the output of
        encoder layer `out_layer_idx` as a dense Seq (B, T, model_dim) whose lens are the padding-mask frame counts, and
        the number of frames per row that carry a unit (frames of the collated sequence).  marks (timing tools): four CUDA
        events recorded after the front kernel, the conv stack, the projection + positional conv and the layers."""
        def mark(i):
            if marks is not None:
                marks[i].record()

        cfg, M = self.cfg, self.M
        if not 0 <= out_layer_idx < cfg.num_encoder_layers:
            raise ValueError(f"out_layer_idx {out_layer_idx} is outside [0, {cfg.num_encoder_layers})")
        num_samples = [int(n) for n in num_samples]
        self.check_batch(num_samples)
        B, dev = len(num_samples), self.device
        per_layer, mask = self.frame_counts(num_samples)
        n_out = [pl[-1] for pl in per_layer]
        if wave.shape[1] < max(num_samples):
            raise ValueError(f"wave has {wave.shape[1]} columns, fewer than the longest row's {max(num_samples)} samples")
        wave = wave.to(dev, torch.float32)
        if wave.stride(1) != 1:
            wave = wave.contiguous()
        ns = torch.tensor(num_samples, dtype=I32, device=dev)
        Tp = (max(pl[0] for pl in per_layer) + 63) // 64 * 64
        x = ops.w2v2_front(wave, ns, self.w["fe0.w"], self.w["fe0.b"], self.w[f"{self._fe(0)}.w"], self.w[f"{self._fe(0)}.b"], Tp)
        mark(0)
        for i, (_, k, _) in enumerate(self.descs[1:], 1):
            lens = torch.tensor([pl[i] for pl in per_layer], dtype=I32, device=dev)
            pairs = Seq(B, Tp // 2, 1024, buf=x.buf.view(B * Tp // 2, 1024))
            y = ops.gemm(pairs, self.w[f"fe{i}.w"], 512, self.w[f"fe{i}.b"], taps=2 if k == 3 else 1)
            Tp //= 2
            x = ops.layernorm_gelu(Seq(B, Tp, 512, lens=lens, buf=y.buf), self.w[f"{self._fe(i)}.w"], self.w[f"{self._fe(i)}.b"])
        mark(1)
        # post-extract LayerNorm into blocks with >= K/2 zero rows after every sequence, projection with padded frames zeroed
        T = max(n_out)
        half = cfg.pos_conv_kernel_size // 2
        Te = (T + half + 7) // 8 * 8
        mask_lens = torch.tensor(mask, dtype=I32, device=dev)
        xe = Seq(B, Te, 512, rows=Te, lens=mask_lens, zero=True)
        ops.layernorm(Seq(B, Tp, 512, lens=mask_lens, buf=x.buf), self.w["encoder_frontend.post_extract_layer_norm.w"],
                      self.w["encoder_frontend.post_extract_layer_norm.b"], out=Seq(B, Tp, 512, rows=Te, buf=xe.buf), mask=True)
        xe = ops.gemm(xe, self.w["encoder_frontend.model_dim_proj.w"], M, self.w["encoder_frontend.model_dim_proj.b"], mask=True)
        pc = ops.grouped_conv_gelu_res(xe, self.pos_w, self.w["pos.b"], cfg.pos_conv_kernel_size, Seq(B, Te, M, rows=Te, zero=False))
        x = Seq(B, T, M, lens=mask_lens)
        x.buf.view(B, T, M).copy_(pc.buf.view(B, Te, M)[:, :T])
        mark(2)
        for i in range(out_layer_idx + 1):
            x = self._layer(x, f"encoder.layers.{i}")
        mark(3)
        return x, n_out

    def units(self, feats: Seq, n_out: Sequence[int]) -> List[torch.Tensor]:
        """Nearest centroid of every frame that carries a unit: a list of B int64 tensors of n_out[b] units."""
        lens = torch.tensor(list(n_out), dtype=I32, device=self.device)
        x = Seq(feats.B, feats.T, feats.C, rows=feats.Tp, buf=feats.buf)
        u = ops.nearest_centroid(x, self.w["km.c"], self.w["km.nhn"], lens).view(feats.B, feats.Tp)
        return [u[b, :n_out[b]].long() for b in range(feats.B)]

    @staticmethod
    def _fe(i: int) -> str:
        return f"encoder_frontend.feature_extractor.layers.{i}.layer_norm"

    def _layer(self, x: Seq, p: str) -> Seq:
        M, w = self.M, self.w
        h = ops.layernorm(x, w[p + ".self_attn_layer_norm.w"], w[p + ".self_attn_layer_norm.b"])
        qkv = ops.gemm(h, w[p + ".qkv.w"], 3 * M, w[p + ".qkv.b"])
        a = Seq(x.B, x.T, M, lens=x.lens)
        b = qkv.buf
        ops.attention_hd80(b[:, :M], b[:, M:2 * M], b[:, 2 * M:], a.buf, x.B, self.H, x.T, x.T, x.Tp, 0, x.Tp, 0, x.lens)
        x = ops.gemm(a, w[p + ".self_attn.output_proj.w"], M, w[p + ".self_attn.output_proj.b"], res1=x)
        h = ops.layernorm(x, w[p + ".ffn_layer_norm.w"], w[p + ".ffn_layer_norm.b"])
        t = ops.gemm(h, w[p + ".ffn.inner_proj.w"], self.cfg.ffn_inner_dim, w[p + ".ffn.inner_proj.b"], act=ACT_GELU)
        return ops.gemm(t, w[p + ".ffn.output_proj.w"], M, w[p + ".ffn.output_proj.b"], res1=x)
