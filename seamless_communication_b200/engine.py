"""Host-side orchestration of the S2ST hot path on top of the C-ABI kernels.

`UnitYEngine` holds the packed device weights of a UnitY2 model (speech encoder + adaptor, NLLB text decoder, NAR
T2U) and sequences the kernels for each module of the path; `VocoderEngine` does the same for Code-HiFiGAN.
Reference call stack being replaced: SURVEY.md 3.1 (inference/translator.py:216 -> inference/generator.py:228 ->
models/unity/model.py / fairseq2 modules -> models/vocoder/*).

Weight packing (one-time, at load):
  * Linear weights stay (out,in) fp16 (K-major B operand of the wgmma GEMM); biases and LayerNorm params fp32;
  * q/k/v projections are concatenated into one (3M,M) matrix; cross-attention k/v into (2M,M);
  * Conv1d (out,in,k) -> (out,k,in) so that K index = tap*C_in + c matches the TMA tap walk;
  * GLU-feeding weights are row-interleaved (a_j, b_j) so the GEMM epilogue can gate adjacent accumulator columns;
  * HiFi-GAN weight_norm is folded (g*v/||v||), ConvTranspose1d becomes a 3-tap GEMM with stride*C_out outputs.
"""
from __future__ import annotations

import collections
import threading
import ctypes as C
import math
import os
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib, ops
from ._lib import BeamDesc, check
from .config import UnitYConfig, VocoderConfig
from .ops import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_SILU, F16, Seq

I32 = torch.int32
_CAPTURE_LOCK = threading.Lock()


def _capture_stream() -> Optional[torch.cuda.Stream]:
    """The stream a step graph is captured on: the calling thread's own stream when it has one (a LanePool lane), else
    torch's capture stream.  torch hands its pool's 32 streams out round-robin, so a capture stream shared by every thread
    can be another lane's stream, and that lane's work would then run inside the capture."""
    cur = torch.cuda.current_stream()
    return None if cur == torch.cuda.default_stream(cur.device) else cur


def sinusoid_table(max_len: int, dim: int, legacy_pad_idx: int = 1) -> torch.Tensor:
    """SinusoidalPositionEncoder table ([fs2-recall], oracle/ASSUMPTIONS.md #4; slice mirrored fairseq2.cpp:900-915)."""
    half = dim // 2
    steps = torch.arange(1 + legacy_pad_idx, 1 + legacy_pad_idx + max_len, dtype=torch.float32)
    inv = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000.0) / (half - 1)))
    ang = steps[:, None] * inv[None, :]
    return torch.cat([torch.sin(ang), torch.cos(ang)], dim=1).contiguous()


XL_POS_CTX = 4096  # rows n_ctx-1 +- (n_ctx-1) of w2v-BERT v1's relative position table (fairseq2.cpp:622)


def relpos_table(n_ctx: int, dim: int) -> torch.Tensor:
    """RelativePositionalEncoding table of w2v-BERT v1, (2*n_ctx-1, dim) fp32 ([fs2-recall]; DESIGN.md §8): row r encodes
    the step n_ctx-1-r (rows 0..n_ctx-1: steps n_ctx-1 .. 0, the rest -1 .. -(n_ctx-1)); column 2i holds
    sin(step * exp(-2i ln(1e4) / dim)), column 2i+1 the cosine.  A checkpoint's `speech_encoder.pos_enc` replaces it."""
    steps = torch.arange(n_ctx - 1, -n_ctx, -1, dtype=torch.float32)
    inv = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    ang = steps[:, None] * inv[None, :]
    return torch.stack([torch.sin(ang), torch.cos(ang)], dim=2).reshape(2 * n_ctx - 1, dim).contiguous()


def _interleave_glu(w: torch.Tensor) -> torch.Tensor:
    """rows [a_0..a_{M-1}, b_0..b_{M-1}] -> [a_0, b_0, a_1, b_1, ...] (GLU(dim=channels) pairs adjacent)."""
    M = w.shape[0] // 2
    return torch.stack([w[:M], w[M:]], dim=1).reshape(w.shape).contiguous()


class UnitYEngine:
    decode_fused = False  # bench.py reads it for its decoder-step label: every step is the per-op launch chain

    def __init__(self, cfg: UnitYConfig, state_dict: Dict[str, torch.Tensor], tokenizers, device="cuda",
                 decoder_weight_dtype=torch.float16):
        if decoder_weight_dtype not in (torch.float16, torch.float8_e4m3fn):
            raise ValueError(f"decoder_weight_dtype must be torch.float16 or torch.float8_e4m3fn, got {decoder_weight_dtype}")
        _lib.require_cuda()
        self.cfg = cfg
        self.device = torch.device(device)
        self.text_tokenizer, self.char_tokenizer = tokenizers
        self.M, self.H = cfg.model_dim, cfg.num_heads
        assert cfg.head_dim == 64, "attention kernels are specialised for head_dim 64"
        # the NAR T2U (v2) is recognised by its character embedding; an autoregressive T2U (v1) has none, and only its
        # encoder is packed here (its decoder runs on a decoder-only engine of its own, models/unity/model.py)
        self.has_t2u = "t2u_model.decoder_frontend.embed_char.weight" in state_dict
        self.has_t2u_encoder = "t2u_model.encoder.layer_norm.weight" in state_dict
        self.has_encoder = any(k.startswith("speech_encoder.") for k in state_dict)  # a monotonic text decoder has none
        # FP8 decoder weights (models/fp8_weights.py): the decoder's products and the tied projection read e4m3 weights
        # with per-feature scales, and every fp16 copy of those weights holds W' = q * scale, so every path computes the
        # same model
        self.fp8 = decoder_weight_dtype == torch.float8_e4m3fn
        q8 = self._quantize_decoder(state_dict) if self.fp8 else None
        if q8 is not None:
            from .models.fp8_weights import dequantize_rows
            state_dict = dict(state_dict)
            for k, (q, s) in q8.items():
                state_dict[k] = dequantize_rows(q, s)
        self._pack(state_dict)
        if q8 is not None:
            self._pack_e4m3(q8)
        self.pos = sinusoid_table(cfg.max_seq_len, self.M).to(self.device)
        if self.has_t2u:
            self._build_char_tables()
        self._graphs = collections.OrderedDict()
        # lanes (parallel.LanePool): several host threads drive independent batches on their own streams; each thread
        # sees its own search states / graphs (the lane is part of the cache key) and its own "last search" record
        self._tls = threading.local()
        self._count_lock = threading.Lock()
        self._state_lock = threading.RLock()
        # L2 prefetch of the next decoder-step GEMM's weights: only without programmatic dependent launch.  With PDL the
        # next GEMM's CTAs start under their predecessor and load their own first weight tiles, and with several lanes
        # in flight the extra bulk prefetches only evict the other lanes' data (DESIGN section 5)
        pdl = _lib.load().sb_pdl_enabled() != 0
        self.decode_prefetch = os.environ.get("SB_DECODE_PREFETCH", "0" if pdl else "1") != "0"
        self.graph_kernels = 0  # kernels executed through CUDA-graph replays (bench.py: gpu_launches)
        # all six weight products of a decoder step on the transposed wgmma kernel (decode_gemm.cu) at <= 256 rows;
        # SB_DECODE_GEMM_T=0 selects the row-major wgmma chain instead
        self.decode_gemm_t = os.environ.get("SB_DECODE_GEMM_T", "1") != "0"
        self.topk_tiles = os.environ.get("SB_TOPK_TILES", "1") != "0"  # top-K from the projection's per-tile statistics

    # ------------------------------------------------------------------------------------------ weight packing
    def _pack(self, sd):
        dev = self.device
        w: Dict[str, torch.Tensor] = {}

        def h(t):
            return t.to(dev, F16).contiguous()

        def f(t):
            return t.to(dev, torch.float32).contiguous()

        def lin(name):
            w[name + ".w"] = h(sd[name + ".weight"])
            if name + ".bias" in sd:
                w[name + ".b"] = f(sd[name + ".bias"])

        def ln(name):
            w[name + ".w"], w[name + ".b"] = f(sd[name + ".weight"]), f(sd[name + ".bias"])

        def conv(name, glu=False):
            cw = sd[name + ".weight"].permute(0, 2, 1).reshape(sd[name + ".weight"].shape[0], -1)  # (out, k*in)
            cb = sd.get(name + ".bias")
            if glu:
                cw = _interleave_glu(cw)
                cb = _interleave_glu(cb) if cb is not None else None
            w[name + ".w"] = h(cw)
            if cb is not None:
                w[name + ".b"] = f(cb)

        def mha(name, fuse_qkv=True):
            if fuse_qkv:
                w[name + ".qkv.w"] = h(torch.cat([sd[f"{name}.{p}_proj.weight"] for p in "qkv"], 0))
                w[name + ".qkv.b"] = f(torch.cat([sd[f"{name}.{p}_proj.bias"] for p in "qkv"], 0))
            else:
                lin(name + ".q_proj")
                w[name + ".kv.w"] = h(torch.cat([sd[f"{name}.{p}_proj.weight"] for p in "kv"], 0))
                w[name + ".kv.b"] = f(torch.cat([sd[f"{name}.{p}_proj.bias"] for p in "kv"], 0))
            lin(name + ".output_proj")

        c = self.cfg
        v1 = c.encoder_variant == "v1"
        if self.has_encoder:
            ln("speech_encoder_frontend.post_extract_layer_norm")
            lin("speech_encoder_frontend.model_dim_proj")
        for i in range(c.enc_layers if self.has_encoder else 0):
            p = f"speech_encoder.inner.layers.{i}"
            for n in ("ffn1", "ffn2"):
                ln(f"{p}.{n}_layer_norm"); lin(f"{p}.{n}.inner_proj"); lin(f"{p}.{n}.output_proj")
            ln(f"{p}.self_attn_layer_norm"); mha(f"{p}.self_attn")
            dw = sd[f"{p}.conv.depthwise_conv.weight"].reshape(c.model_dim, c.dw_kernel)
            if v1:
                # u is folded into the q projection's bias (q + u is what multiplies k); the kernel adds v - u for the
                # positional term.  R = r_proj(pos table) is one GEMM per call (encode_speech).
                a = sd[f"{p}.self_attn.sdpa.u_bias"].double().reshape(-1)
                w[f"{p}.self_attn.qkv.b"][:self.M] += a.to(dev, torch.float32)
                w[f"{p}.r_proj.w"] = h(sd[f"{p}.self_attn.sdpa.r_proj.weight"])
                w[f"{p}.vu"] = f((sd[f"{p}.self_attn.sdpa.v_bias"].double().reshape(-1) - a).reshape(self.H, -1))
                # eval BatchNorm folded in fp64: w' = w * g / sqrt(var + eps), bias = beta - mean * g / sqrt(var + eps)
                bn = f"{p}.conv.batch_norm"
                scale = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + 1e-5)
                w[f"{p}.conv.dw.w"] = h(dw.double() * scale[:, None])
                w[f"{p}.conv.bn.b"] = f(sd[bn + ".bias"].double() - sd[bn + ".running_mean"].double() * scale)
            else:
                w[f"{p}.rel_k"] = h(sd[f"{p}.self_attn.sdpa.rel_k_embed.weight"])
                w[f"{p}.conv.dw.w"] = h(dw)
                ln(f"{p}.conv.layer_norm")
            ln(f"{p}.conv_layer_norm")
            conv(f"{p}.conv.pointwise_conv1", glu=True)
            conv(f"{p}.conv.pointwise_conv2")
            ln(f"{p}.layer_norm")
        if self.has_encoder and v1:
            pe = sd.get("speech_encoder.pos_enc")
            if pe is None:
                pe = relpos_table(XL_POS_CTX, c.model_dim)
            elif tuple(pe.shape) != (2 * XL_POS_CTX - 1, c.model_dim):
                raise ValueError(f"speech_encoder.pos_enc has shape {tuple(pe.shape)}, expected {(2 * XL_POS_CTX - 1, c.model_dim)}")
            w["relpos"] = h(pe)
        if self.has_encoder:
            ln("speech_encoder.inner_layer_norm"); lin("speech_encoder.proj1"); lin("speech_encoder.proj2")
            p = "speech_encoder.adaptor_layers.0"
            ln(f"{p}.residual_layer_norm"); conv(f"{p}.residual_conv", glu=True)
            ln(f"{p}.self_attn_layer_norm"); conv(f"{p}.self_attn_conv", glu=True)
            mha(f"{p}.self_attn"); ln(f"{p}.ffn_layer_norm"); lin(f"{p}.ffn.inner_proj"); lin(f"{p}.ffn.output_proj")
            ln("speech_encoder.layer_norm")
        w["text_embed"] = h(sd["text_decoder_frontend.embed.weight"])  # tied with final_proj (builder.py:451)
        for i in range(c.dec_layers):
            p = f"text_decoder.layers.{i}"
            ln(f"{p}.self_attn_layer_norm"); mha(f"{p}.self_attn")
            ln(f"{p}.encoder_decoder_attn_layer_norm"); mha(f"{p}.encoder_decoder_attn", fuse_qkv=False)
            ln(f"{p}.ffn_layer_norm"); lin(f"{p}.ffn.inner_proj"); lin(f"{p}.ffn.output_proj")
        ln("text_decoder.layer_norm")
        if self.has_t2u_encoder:
            for i in range(c.t2u_enc_layers):
                p = f"t2u_model.encoder.layers.{i}"
                ln(f"{p}.self_attn_layer_norm"); mha(f"{p}.self_attn")
                ln(f"{p}.ffn_layer_norm"); lin(f"{p}.ffn.inner_proj"); lin(f"{p}.ffn.output_proj")
            ln("t2u_model.encoder.layer_norm")
        if self.has_t2u:
            P = "t2u_model.decoder_frontend"
            w["unit_embed"] = h(sd[P + ".embed.weight"])
            w["char_embed"] = h(sd[P + ".embed_char.weight"])
            w["alpha"] = f(sd[P + ".pos_emb_alpha"]); w["alpha_char"] = f(sd[P + ".pos_emb_alpha_char"])
            dp = P + ".variance_adaptor.duration_predictor"
            conv(dp + ".conv1.0"); ln(dp + ".ln1"); conv(dp + ".conv2.0"); ln(dp + ".ln2")
            w[dp + ".proj.w"] = h(sd[dp + ".proj.weight"].reshape(-1))
            self.dur_bias = float(sd[dp + ".proj.bias"][0])
            for i in range(c.t2u_dec_layers):
                p = f"t2u_model.decoder.layers.{i}"
                mha(f"{p}.self_attn"); ln(f"{p}.self_attn_layer_norm")
                conv(f"{p}.conv1d.conv1"); conv(f"{p}.conv1d.conv2"); ln(f"{p}.conv1d_layer_norm")
            ln("t2u_model.decoder.layer_norm")
        self.w = w

    def _quantize_decoder(self, sd):
        """{state-dict name: (q e4m3, scale fp32)} on the device for every weight FP8 mode quantizes."""
        from .models.fp8_weights import decoder_weight_names, quantize_rows
        return {k: quantize_rows(sd[k].to(self.device)) for k in decoder_weight_names(sd, self.cfg)}

    def _pack_e4m3(self, q8):
        """The e4m3 weights and scales of the decoder step beside the fp16 ones: `<name>.q8` (n, K) float8_e4m3fn and
        `<name>.s` (n,) fp32, q|k|v concatenated as their fp16 copies are."""
        w = self.w

        def put(key, names):
            w[key + ".q8"] = torch.cat([q8[n][0] for n in names]).contiguous()
            w[key + ".s"] = torch.cat([q8[n][1] for n in names]).contiguous()

        put("text_embed", ["text_decoder_frontend.embed.weight"])
        for i in range(self.cfg.dec_layers):
            p = f"text_decoder.layers.{i}"
            put(p + ".self_attn.qkv", [f"{p}.self_attn.{x}_proj.weight" for x in "qkv"])
            for n in ("self_attn.output_proj", "encoder_decoder_attn.q_proj", "encoder_decoder_attn.output_proj",
                      "ffn.inner_proj", "ffn.output_proj"):
                put(f"{p}.{n}", [f"{p}.{n}.weight"])

    def _build_char_tables(self):
        """Per-token tables replacing the Python string loops of nar_decoder_frontend.py:130-259."""
        tok, ctok = self.text_tokenizer, self.char_tokenizer
        V = self.cfg.text_vocab
        pieces = [tok.model.index_to_token(i) for i in range(V)]
        max_chars = max(len(p) for p in pieces)
        tl = torch.zeros(V, dtype=torch.uint8)
        fl = torch.zeros(V, dtype=torch.uint8)
        tc = torch.zeros(V, max_chars, dtype=torch.int32)
        SP = "▁"
        cache: Dict[str, int] = {}
        for i, p in enumerate(pieces):
            tl[i] = len(p)
            punc = len(p) == 1 and not p.isalpha() and not p.isnumeric() and p != SP
            nss = len(p) > 1 and p[0] == SP
            fl[i] = int(punc) | (int(nss) << 1)
            for j, ch in enumerate(p):
                if ch not in cache:
                    cache[ch] = ctok.model.token_to_index(ch)
                tc[i, j] = cache[ch]
        self.tok_len, self.tok_flags, self.tok_chars = tl.to(self.device), fl.to(self.device), tc.to(self.device)
        self.max_chars = max_chars

    # ------------------------------------------------------------------------------------------ building blocks
    def _lin(self, x: Seq, name: str, n: int, **kw) -> Seq:
        return ops.gemm(x, self.w[name + ".w"], n, self.w.get(name + ".b"), **kw)

    def _ln(self, x: Seq, name: str, **kw) -> Seq:
        return ops.layernorm(x, self.w[name + ".w"], self.w[name + ".b"], **kw)

    def _mha_self(self, x_in: Seq, name: str, res: Seq, *, causal=False, rel=None) -> Seq:
        M = self.M
        qkv = self._lin(x_in, name + ".qkv", 3 * M)
        c = self.cfg
        a = ops.self_attention(qkv, self.H, causal=causal, rel_k=rel, rel_left=c.shaw_left if rel is not None else 0,
                               rel_right=c.shaw_right if rel is not None else 0)
        return self._lin(a, name + ".output_proj", M, res1=res)

    def _ffn(self, x_in: Seq, name: str, inner: int, act: int, res: Seq, alpha=1.0) -> Seq:
        t = self._lin(x_in, name + ".inner_proj", inner, act=act)
        return self._lin(t, name + ".output_proj", self.M, res1=res, alpha=alpha)

    # ------------------------------------------------------------------------------------------ a3-a6 speech encoder
    @torch.inference_mode()
    def encode_speech(self, fbank: torch.Tensor, lens: Optional[torch.Tensor], return_inner=False):
        """fbank (B, T_fb, 80) fp16 cuda, lens (B,) int32 cuda or None -> encoder output Seq (B, S_a, M), lens."""
        if not self.has_encoder:
            raise RuntimeError("this engine was built without a speech encoder (text-decoder-only state dict)")
        c, M = self.cfg, self.M
        B, T_fb, Cf = fbank.shape
        s = c.fbank_stride
        T2 = T_fb - (T_fb % s)
        if T2 != T_fb:
            fbank = fbank[:, :T2].contiguous()
            lens = torch.clamp(lens, max=T2) if lens is not None else None
        S = T2 // s
        v1 = c.encoder_variant == "v1"
        if v1 and S > XL_POS_CTX:  # the relative position table holds distances up to n_ctx - 1
            raise ValueError(f"The input sequence length must be less than or equal to the maximum sequence length "
                             f"({XL_POS_CTX}), but is {S} instead.")
        lens_s = (lens // s).to(I32) if lens is not None else None
        x = Seq(B, S, Cf * s, lens=lens_s, buf=fbank.reshape(B * S, Cf * s))
        x = self._ln(x, "speech_encoder_frontend.post_extract_layer_norm")
        x = self._lin(x, "speech_encoder_frontend.model_dim_proj", M)
        for i in range(c.enc_layers):
            p = f"speech_encoder.inner.layers.{i}"
            x = self._ffn(self._ln(x, p + ".ffn1_layer_norm"), p + ".ffn1", c.enc_ffn_dim, ACT_SILU, x, alpha=0.5)
            if v1:
                # R = r_proj(table rows n_ctx-S .. n_ctx+S-2), shared by the batch; row S-1+j-i encodes distance i-j
                pos = Seq(1, 2 * S - 1, M, buf=self.w["relpos"][XL_POS_CTX - S:XL_POS_CTX + S - 1])
                r = self._lin(pos, p + ".r_proj", M)
                qkv = self._lin(self._ln(x, p + ".self_attn_layer_norm"), p + ".self_attn.qkv", 3 * M)
                a = ops.self_attention_relpos(qkv, self.H, r.buf, vb=self.w[p + ".vu"])
                x = self._lin(a, p + ".self_attn.output_proj", M, res1=x)
            else:
                x = self._mha_self(self._ln(x, p + ".self_attn_layer_norm"), p + ".self_attn", x, rel=self.w[p + ".rel_k"])
            hcv = self._ln(x, p + ".conv_layer_norm", mask=True)
            g = self._lin(hcv, p + ".conv.pointwise_conv1", 2 * M, glu=True)
            if v1:
                d = ops.dwconv_bias_silu(g, self.w[p + ".conv.dw.w"], self.w[p + ".conv.bn.b"], c.dw_kernel)
            else:
                d = ops.dwconv_ln_silu(g, self.w[p + ".conv.dw.w"], self.w[p + ".conv.layer_norm.w"],
                                       self.w[p + ".conv.layer_norm.b"], c.dw_kernel)
            x = self._lin(d, p + ".conv.pointwise_conv2", M, res1=x)
            x = self._ffn(self._ln(x, p + ".ffn2_layer_norm"), p + ".ffn2", c.enc_ffn_dim, ACT_SILU, x, alpha=0.5)
            x = self._ln(x, p + ".layer_norm")
        inner = x
        x = self._ln(x, "speech_encoder.inner_layer_norm")
        t = self._lin(x, "speech_encoder.proj1", 4 * M, act=ACT_RELU)
        x = self._lin(t, "speech_encoder.proj2", M, res1=x, alpha=0.5)
        # adaptor layer (adaptor_block.py:236-314): Conv1d(k, stride k... here k == stride) as a reshaped GEMM
        p = "speech_encoder.adaptor_layers.0"
        k, st = c.adaptor_kernel, c.adaptor_stride
        assert k == st, "adaptor conv is lowered to a reshape GEMM and needs kernel == stride"
        S_a = S // st + 1
        lens_a = (lens_s // st + 1).to(I32) if lens_s is not None else None

        S_used = min(S, st * S_a - k // 2)  # frames past the last conv window are never read (floor in the length formula)
        x_used = Seq(B, S_used, M, x.PH, x.Tp, lens_s, buf=x.buf)

        def pooled(ln_name, conv_name):
            padded = Seq(B, S_used, M, halo=k // 2, rows=st * S_a, lens=lens_s)  # left pad k//2, zero right pad
            self._ln(x_used, ln_name, out=padded)
            view = Seq(B, S_a, st * M, lens=lens_a, buf=padded.buf.view(B * S_a, st * M))
            return ops.gemm(view, self.w[conv_name + ".w"], 2 * M, self.w[conv_name + ".b"], glu=True)

        residual = pooled(p + ".residual_layer_norm", p + ".residual_conv")
        hh = pooled(p + ".self_attn_layer_norm", p + ".self_attn_conv")
        hh = self._mha_self(hh, p + ".self_attn", residual)
        hh = self._ffn(self._ln(hh, p + ".ffn_layer_norm"), p + ".ffn", c.enc_ffn_dim, ACT_RELU, hh)
        out = self._ln(hh, "speech_encoder.layer_norm")
        return (out, lens_a, inner) if return_inner else (out, lens_a)

    # ------------------------------------------------------------------------------------------ a7-a9 beam search
    def _cross_kv(self, enc: Seq):
        """per-utterance static cross-attention K/V for every decoder layer (computed once, not per beam)."""
        return [self._lin(enc, f"text_decoder.layers.{i}.encoder_decoder_attn.kv", 2 * self.M)
                for i in range(self.cfg.dec_layers)]

    def _decoder_step_forward(self, st, record=False):
        """One incremental decoder step for R rows; all shapes static, step index read from st['step'] on device.
        The three residual GEMMs of a layer (self-attn out, cross-attn out, FFN out) run split-K so that all SMs stream
        weights even at M = R rows, and their reduction (+bias, +residual) is fused into the LayerNorm that follows.
        `record`: the last layer's head-summed cross-attention weights go to st["attn_hist"][step] (token timestamps)."""
        lib = _lib.load()
        c, M, H = self.cfg, self.M, self.H
        R, stream = st["R"], ops._stream()
        x, h, part = st["x"], st["h"], st["partials"]
        w = self.w
        check(lib.sb_embed_step(st["seqs"].data_ptr(), st["ML"], st["step"].data_ptr(), w["text_embed"].data_ptr(),
                                self.pos.data_ptr(), math.sqrt(M), x.buf.data_ptr(), R, M, stream), "sb_embed_step")
        self._ln(x, "text_decoder.layers.0.self_attn_layer_norm", out=h)
        S_ATT, S_FFN, S_QKV, SR = st["splits_attn"], st["splits_ffn"], st["splits_qkv"], ops.slice_rows(R)
        pf = self.decode_prefetch  # each GEMM pulls the weights of the GEMM after it into L2 (latency-bound chain)
        f8 = self.fp8  # e4m3 weights: every product on the e4m3 entries, at any row count

        def splitk(a, name, n, splits, part, nxt):
            if f8:
                ops.gemm_splitk_e4m3(a, w[name + ".q8"], w[name + ".s"], n, splits, part,
                                     prefetch=w[nxt + ".q8"] if pf and nxt else None)
            else:
                ops.gemm_splitk(a, w[name + ".w"], n, splits, part, prefetch=w[nxt + ".w"] if pf and nxt else None,
                                transposed=st["gemm_t"])

        for i in range(c.dec_layers):
            p = f"text_decoder.layers.{i}"
            last = i + 1 == c.dec_layers
            nxt = "text_decoder.layer_norm" if last else f"text_decoder.layers.{i + 1}.self_attn_layer_norm"
            w_next = None if last else f"text_decoder.layers.{i + 1}.self_attn.qkv"
            # qkv / q projections also run split-K; their partials are reduced (+bias) inside the attention kernels
            splitk(h, p + ".self_attn.qkv", 3 * M, S_QKV, st["part_qkv"], p + ".self_attn.output_proj")
            check(lib.sb_decode_self_attn(None, st["part_qkv"].data_ptr(), S_QKV, SR, w[p + ".self_attn.qkv.b"].data_ptr(),
                                          st["kc"][i].data_ptr(), st["vc"][i].data_ptr(), st["anc"].data_ptr(), st["ML"],
                                          st["step"].data_ptr(), st["ML"], st["att"].buf.data_ptr(), R, H, stream),
                  "sb_decode_self_attn")
            splitk(st["att"], p + ".self_attn.output_proj", M, S_ATT, part, p + ".encoder_decoder_attn.q_proj")
            ops.splitk_reduce_ln(part, S_ATT, w[p + ".self_attn.output_proj.b"], x, w[p + ".encoder_decoder_attn_layer_norm.w"],
                                 w[p + ".encoder_decoder_attn_layer_norm.b"], h)
            splitk(h, p + ".encoder_decoder_attn.q_proj", M, S_ATT, part, p + ".encoder_decoder_attn.output_proj")
            kv = st["cross_kv"][i].buf
            check(lib.sb_decode_cross_attn(None, part.data_ptr(), S_ATT, SR, w[p + ".encoder_decoder_attn.q_proj.b"].data_ptr(),
                                           kv.data_ptr(), kv[:, M:].data_ptr(), kv.stride(0), ops._p(st["enc_lens"]),
                                           st["S_enc"], st["att"].buf.data_ptr(), R, st["beam"], H, stream),
                  "sb_decode_cross_attn")
            if record and last:  # reads the q partials before the next product overwrites them
                ops.decode_cross_attn_weights(part, S_ATT, SR, w[p + ".encoder_decoder_attn.q_proj.b"], kv, st["enc_lens"],
                                              st["S_enc"], st["step"], st["attn_hist"], R, st["beam"], H)
            splitk(st["att"], p + ".encoder_decoder_attn.output_proj", M, S_ATT, part, p + ".ffn.inner_proj")
            ops.splitk_reduce_ln(part, S_ATT, w[p + ".encoder_decoder_attn.output_proj.b"], x, w[p + ".ffn_layer_norm.w"],
                                 w[p + ".ffn_layer_norm.b"], h)
            if f8:
                t = ops.gemm_decode_e4m3(h, w[p + ".ffn.inner_proj.q8"], w[p + ".ffn.inner_proj.s"], c.dec_ffn_dim,
                                         w[p + ".ffn.inner_proj.b"], act=ACT_RELU, out=st["ffn"],
                                         prefetch=w[p + ".ffn.output_proj.q8"] if pf else None)
            elif st["gemm_t"]:
                t = ops.gemm_decode(h, w[p + ".ffn.inner_proj.w"], c.dec_ffn_dim, w[p + ".ffn.inner_proj.b"], act=ACT_RELU,
                                    out=st["ffn"], prefetch=w[p + ".ffn.output_proj.w"] if pf else None)
            else:
                t = self._lin(h, p + ".ffn.inner_proj", c.dec_ffn_dim, act=ACT_RELU, out=st["ffn"],
                              prefetch=w[p + ".ffn.output_proj.w"] if pf else None)
            splitk(t, p + ".ffn.output_proj", M, S_FFN, part, w_next)
            ops.splitk_reduce_ln(part, S_FFN, w[p + ".ffn.output_proj.b"], x, w[nxt + ".w"], w[nxt + ".b"], h)
        check(lib.sb_store_step(h.buf.data_ptr(), st["hist"].data_ptr(), st["step"].data_ptr(), R * M * 2, stream), "sb_store_step")
        if f8:
            ops.vocab_proj_e4m3(h, w["text_embed.q8"], w["text_embed.s"], c.text_vocab, st["logits"], st["tile_stats"])
        else:
            ops.gemm(h, w["text_embed"], c.text_vocab, None, out=st["logits"], out_f32=True, tile_stats=st["tile_stats"])

    def _topk(self, st, eos_idx, unk_penalty, bans=None):
        """log-softmax statistics + top-K candidates of every row (st["logits"] / st["tile_stats"] of the last projection).
        `bans`: a ban-list buffer of the state (st["ban"] or st["ngram"]); the ids written to its `ids` / `n` are not
        candidates."""
        lib, c = _lib.load(), self.cfg
        if bans is not None:
            b = bans
            if st["tile_stats"] is not None:
                check(lib.sb_logits_topk_tiles_ban(st["logits"].buf.data_ptr(), st["logits"].buf.stride(0), st["tile_stats"].data_ptr(),
                                                   st["R"], c.text_vocab, c.text_pad, eos_idx, c.text_unk, unk_penalty, st["K"],
                                                   st["cand_val"].data_ptr(), st["cand_idx"].data_ptr(), st["eos_lprob"].data_ptr(),
                                                   b["ids"].data_ptr(), b["n"].data_ptr(), b["cap"], ops._stream()),
                      "sb_logits_topk_tiles_ban")
            else:
                check(lib.sb_logits_topk_ban(st["logits"].buf.data_ptr(), st["logits"].buf.stride(0), st["R"], c.text_vocab, c.text_pad,
                                             eos_idx, c.text_unk, unk_penalty, st["K"], st["cand_val"].data_ptr(),
                                             st["cand_idx"].data_ptr(), st["eos_lprob"].data_ptr(), b["ids"].data_ptr(),
                                             b["n"].data_ptr(), b["cap"], ops._stream()), "sb_logits_topk_ban")
            return
        if st["tile_stats"] is not None:
            check(lib.sb_logits_topk_tiles(st["logits"].buf.data_ptr(), st["logits"].buf.stride(0), st["tile_stats"].data_ptr(), st["R"],
                                           c.text_vocab, c.text_pad, eos_idx, c.text_unk, unk_penalty, st["K"], st["cand_val"].data_ptr(),
                                           st["cand_idx"].data_ptr(), st["eos_lprob"].data_ptr(), ops._stream()), "sb_logits_topk_tiles")
        else:
            check(lib.sb_logits_topk(st["logits"].buf.data_ptr(), st["logits"].buf.stride(0), st["R"], c.text_vocab, c.text_pad,
                                     eos_idx, c.text_unk, unk_penalty, st["K"], st["cand_val"].data_ptr(),
                                     st["cand_idx"].data_ptr(), st["eos_lprob"].data_ptr(), ops._stream()), "sb_logits_topk")

    def _decoder_step_select(self, st, ban=False, ngram=0):
        """`ban`: banned sequences (sb_ban_step on st["ban"]); `ngram` > 0: n-gram repeat blocking of that size
        (sb_ngram_ban_step on st["ngram"]).  Either feeds the ban-aware top-K."""
        lib = _lib.load()
        stream = ops._stream()
        bans = None
        if ban:
            b = bans = st["ban"]
            check(lib.sb_ban_step(st["seqs"].data_ptr(), st["ML"], st["step"].data_ptr(), st["R"], b["table"].data_ptr(), b["cap"],
                                  b["width"], b["ids"].data_ptr(), b["n"].data_ptr(), stream), "sb_ban_step")
        elif ngram:
            bans = st["ngram"]
            ops.ngram_ban_step(st["seqs"], st["step"], ngram, bans["ids"], bans["n"])
        self._topk(st, self.cfg.text_eos, st["unk_penalty"], bans=bans)
        check(lib.sb_beam_step(C.byref(st["beam_desc"]), stream), "sb_beam_step")
        check(lib.sb_step_advance(st["step"].data_ptr(), stream), "sb_step_advance")

    @property
    def lane(self) -> int:
        return getattr(self._tls, "lane", 0)

    def set_lane(self, lane: int):
        """Bind the calling host thread to search-state lane `lane` (parallel.LanePool calls this once per worker)."""
        self._tls.lane = int(lane)

    @property
    def _last_search_state(self):
        return getattr(self._tls, "last_state", None)

    @_last_search_state.setter
    def _last_search_state(self, st):
        self._tls.last_state = st

    def _search_state(self, B, S_enc, ML, beam, P, has_lens, use_graph):
        with self._state_lock:  # the cache is shared by the lanes' host threads
            return self._search_state_locked(B, S_enc, ML, beam, P, has_lens, use_graph)

    def _search_state_locked(self, B, S_enc, ML, beam, P, has_lens, use_graph):
        """Static buffers + captured CUDA graphs of one decoder step, cached per problem shape so that repeated
        predict() calls replay the same graphs (the reference rebuilds its generator per call, translator.py:179-186;
        construction here stays cheap after the first call)."""
        key = (B, S_enc, ML, beam, P, has_lens, use_graph, self.decode_gemm_t and not self.fp8, self.lane)
        st = self._graphs.get(key)
        if st is not None:
            self._graphs.move_to_end(key)
            return st
        c, M, dev = self.cfg, self.M, self.device
        R = B * beam
        K = min(2 * beam + 1, 16)
        # the top-K kernel returns at most 16 candidates per row and the step needs 2*beam + 1 (one spare for a blocked EOS)
        if 2 * beam + 1 > 16:
            raise ValueError(f"beam_size {beam} is not supported by the top-K kernel (at most 7)")
        st = dict(R=R, ML=ML, beam=beam, K=K, S_enc=S_enc, B=B, P=P, unk_penalty=0.0, key=key)
        st["enc_lens"] = torch.zeros(B, dtype=I32, device=dev) if has_lens else None
        st["cross_kv"] = [Seq(B, S_enc, 2 * M) for _ in range(c.dec_layers)]
        st["seqs"] = torch.zeros((R, ML), dtype=I32, device=dev)
        st["scores"] = torch.zeros((R, ML), dtype=torch.float32, device=dev)
        st["anc"] = torch.zeros((R, ML), dtype=I32, device=dev)
        st["anc_init"] = torch.arange(R, dtype=I32, device=dev)[:, None].repeat(1, ML).contiguous()
        st["step"] = torch.zeros(1, dtype=I32, device=dev)
        st["budget"] = torch.full((1,), ML, dtype=I32, device=dev)  # this search's length budget (<= ML), set per search
        st["kc"] = [torch.empty((ML, R, M), dtype=F16, device=dev) for _ in range(c.dec_layers)]
        st["vc"] = [torch.empty((ML, R, M), dtype=F16, device=dev) for _ in range(c.dec_layers)]
        for name, width in (("x", M), ("h", M), ("q", M), ("att", M), ("qkv", 3 * M), ("ffn", c.dec_ffn_dim)):
            st[name] = Seq(1, R, width)
        st["splits_qkv"], st["splits_attn"], st["splits_ffn"] = ops.decode_splits(R, M, c.dec_ffn_dim)
        # <= 256 rows: all six products run on the transposed wgmma kernel (decode_gemm.cu: the row-major kernel is
        # L2 -> SM bound at these shapes).  It takes the same K slices as the row-major chain: every slice then
        # sums the same k-blocks in the same order, so both paths produce the same partials and the same search.
        st["gemm_t"] = self.decode_gemm_t and R <= 256 and M % 64 == 0 and c.dec_ffn_dim % 64 == 0
        st["part_qkv"] = torch.empty((st["splits_qkv"] * ops.slice_rows(R), 3 * M), dtype=torch.float32, device=dev)
        st["partials"] = torch.empty((max(st["splits_attn"], st["splits_ffn"]) * ops.slice_rows(R), M), dtype=torch.float32,
                                     device=dev)
        st["logits"] = Seq(1, R, c.text_vocab, dtype=torch.float32, buf=torch.empty(
            (R, (c.text_vocab + 7) // 8 * 8), dtype=torch.float32, device=dev))
        # per (128-column tile, row) softmax statistics written by the projection's epilogue (None: two-pass top-K over the logits)
        st["tile_stats"] = (torch.empty(((c.text_vocab + 127) // 128, R, 2), dtype=torch.float32, device=dev)
                            if self.topk_tiles and c.text_vocab >= 128 else None)
        st["cand_val"] = torch.empty((R, K), dtype=torch.float32, device=dev)
        st["cand_idx"] = torch.empty((R, K), dtype=I32, device=dev)
        st["eos_lprob"] = torch.empty((R,), dtype=torch.float32, device=dev)
        fin = dict(count=torch.zeros(B, dtype=I32, device=dev), score=torch.zeros((B, beam), device=dev),
                   len=torch.zeros((B, beam), dtype=I32, device=dev), seqs=torch.zeros((B, beam, ML), dtype=I32, device=dev),
                   active=torch.ones(B, dtype=I32, device=dev), n_active=torch.zeros((1,), dtype=I32, device=dev))
        fin["anc"] = torch.zeros((B, beam, ML), dtype=I32, device=dev)
        fin["scores"] = torch.zeros((B, beam, ML), dtype=torch.float32, device=dev)  # cumulative scores of each finished hypothesis
        st["hist"] = torch.empty((ML, R, M), dtype=F16, device=dev)  # final-LN decoder state of every step
        st["fin"] = fin
        d = BeamDesc()
        d.batch, d.beam, d.max_len, d.vocab, d.K = B, beam, ML, c.text_vocab, K
        d.step_ptr, d.prefix_len, d.eos_idx = st["step"].data_ptr(), P, c.text_eos
        d.cand_val, d.cand_idx, d.eos_lprob = st["cand_val"].data_ptr(), st["cand_idx"].data_ptr(), st["eos_lprob"].data_ptr()
        d.seqs, d.scores, d.anc = st["seqs"].data_ptr(), st["scores"].data_ptr(), st["anc"].data_ptr()
        d.fin_count, d.fin_score, d.fin_len = fin["count"].data_ptr(), fin["score"].data_ptr(), fin["len"].data_ptr()
        d.fin_seqs, d.active, d.n_active = fin["seqs"].data_ptr(), fin["active"].data_ptr(), fin["n_active"].data_ptr()
        d.fin_anc, d.len_budget = fin["anc"].data_ptr(), st["budget"].data_ptr()
        d.fin_scores = fin["scores"].data_ptr()
        st["beam_desc"] = d
        st["g_fwd"] = st["g_sel"] = st["g_sel_ban"] = st["g_fwd_attn"] = st["g_sel_ngram"] = None
        st["n_fwd"] = st["n_sel"] = st["n_sel_ban"] = st["n_fwd_attn"] = st["n_sel_ngram"] = 0
        st["attn_hist"], st["attn_on"] = None, False  # [ML][R][S_enc] fp32, allocated by the first recording search
        st["ban"], st["ban_on"] = None, False
        st["ngram"], st["ngram_on"] = None, 0  # ban lists of n-gram blocking, allocated by the first blocking search
        self._graphs[key] = st
        self._evict_search_states(keep=key)
        return st

    @staticmethod
    def _state_bytes(st) -> int:
        seen, total = set(), 0

        def walk(v):
            nonlocal total
            if isinstance(v, torch.Tensor):
                p = v.untyped_storage().data_ptr()
                if p not in seen:
                    seen.add(p)
                    total += v.untyped_storage().nbytes()
            elif isinstance(v, Seq):
                walk(v.buf)
            elif isinstance(v, dict):
                for x in v.values():
                    walk(x)
            elif isinstance(v, (list, tuple)):
                for x in v:
                    walk(x)
        walk(st)
        return total

    def _evict_search_states(self, keep):
        """The cache is keyed by problem shape (S_enc and max_len follow the audio length), one entry holds the KV caches,
        the history and two CUDA graphs (~4.8 GB at 32 sentences x beam 5): least-recently-used entries are dropped once
        the total exceeds SB_SEARCH_CACHE_GB (default 24 of an 80 GB device), so a service fed variable-length audio cannot grow without
        bound (the reference frees its search state after every call)."""
        budget = float(os.environ.get("SB_SEARCH_CACHE_GB", "24")) * 2 ** 30
        sizes = {k: self._state_bytes(v) for k, v in self._graphs.items()}
        total = sum(sizes.values())
        for k in list(self._graphs.keys()):
            if total <= budget or len(self._graphs) <= 1:
                break
            if k == keep or self._graphs[k] is self._last_search_state:
                continue
            total -= sizes[k]
            del self._graphs[k]

    def _capture(self, st):
        """Capture the forward and the select halves of a decoder step (all pointers/shapes static)."""
        with _CAPTURE_LOCK:  # one capture at a time in the process (launch counting + capture mode are process-wide)
            self._capture_locked(st)

    def _capture_locked(self, st):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):  # eager warm-up: lazy one-time initialisation must not happen during capture
            self._decoder_step_forward(st)
            self._decoder_step_select(st)
        torch.cuda.current_stream().wait_stream(s)
        n0 = ops.launch_count()
        st["g_fwd"] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(st["g_fwd"], stream=_capture_stream(), capture_error_mode="thread_local"):
            self._decoder_step_forward(st)
        n1 = ops.launch_count()
        st["g_sel"] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(st["g_sel"], stream=_capture_stream(), capture_error_mode="thread_local"):
            self._decoder_step_select(st)
        st["n_fwd"], st["n_sel"] = n1 - n0, ops.launch_count() - n1

    def _capture_ban(self, st):
        """Capture the select half with banned sequences (sb_ban_step, ban-aware top-K, sb_beam_step, sb_step_advance) on the
        state's ban table; searches without bans keep replaying g_sel."""
        self._capture_select(st, "g_sel_ban", "n_sel_ban", ban=True)

    def _capture_ngram(self, st):
        """Capture the select half with n-gram repeat blocking of size st["ngram"]["size"] (sb_ngram_ban_step, ban-aware
        top-K, sb_beam_step, sb_step_advance) on the state's ban lists; searches without blocking keep replaying g_sel."""
        self._capture_select(st, "g_sel_ngram", "n_sel_ngram", ngram=st["ngram"]["size"])

    def _capture_select(self, st, graph, count, **kw):
        with _CAPTURE_LOCK:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._decoder_step_select(st, **kw)
            torch.cuda.current_stream().wait_stream(s)
            n0 = ops.launch_count()
            st[graph] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(st[graph], stream=_capture_stream(), capture_error_mode="thread_local"):
                self._decoder_step_select(st, **kw)
            st[count] = ops.launch_count() - n0

    def _capture_attn(self, st):
        """Capture the forward half with the cross-attention weights recorded (sb_decode_cross_attn_weights after the last
        layer's cross-attention); searches that do not record keep replaying g_fwd."""
        with _CAPTURE_LOCK:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._decoder_step_forward(st, record=True)
            torch.cuda.current_stream().wait_stream(s)
            n0 = ops.launch_count()
            st["g_fwd_attn"] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(st["g_fwd_attn"], stream=_capture_stream(), capture_error_mode="thread_local"):
                self._decoder_step_forward(st, record=True)
            st["n_fwd_attn"] = ops.launch_count() - n0

    def _set_bans(self, st, banned):
        """Pack the banned sequences into the state's device table ([count][lengths x cap][cap rows of `width` tokens,
        right-aligned]) with one asynchronous host-to-device copy.  The buffers, and the graph captured on them, are
        replaced only when the table outgrows their capacity (both rounded up to a power of two)."""
        n, width = len(banned), max(len(x) for x in banned)
        b = st["ban"]
        if b is None or n > b["cap"] or width > b["width"]:
            cap = max(16, 1 << (max(n, b["cap"] if b else 0) - 1).bit_length())
            w = max(8, 1 << (max(width, b["width"] if b else 0) - 1).bit_length())
            dev = self.device
            b = st["ban"] = dict(cap=cap, width=w, table=torch.zeros(1 + cap + cap * w, dtype=I32, device=dev),
                                 ids=torch.zeros((st["R"], cap), dtype=I32, device=dev), n=torch.zeros(st["R"], dtype=I32, device=dev))
            st["g_sel_ban"] = None
        cap, w = b["cap"], b["width"]
        host = torch.zeros(1 + cap + cap * w, dtype=I32, pin_memory=True)
        host[0] = n
        lens = host[1:1 + cap]
        toks = host[1 + cap:].view(cap, w)
        for j, seq in enumerate(banned):
            lens[j] = len(seq)
            toks[j, w - len(seq):] = torch.as_tensor(seq, dtype=I32)
        b["table"].copy_(host, non_blocking=True)
        b["host"] = host  # the pinned source stays alive until the copy has run

    def _set_ngram(self, st, n):
        """N-gram blocking of size `n` on this state: ban lists of ML ids per row (a row at step t has at most t-n+2
        starts, t <= ML-1), allocated once per state.  The captured graph has `n` baked in and is recaptured when it
        changes."""
        b = st["ngram"]
        if b is None:
            dev = self.device
            b = st["ngram"] = dict(cap=st["ML"], size=0, ids=torch.zeros((st["R"], st["ML"]), dtype=I32, device=dev),
                                   n=torch.zeros(st["R"], dtype=I32, device=dev))
            with self._state_lock:  # the cache budget now counts the lists too
                self._evict_search_states(keep=st["key"])
        if b["size"] != n:
            b["size"], st["g_sel_ngram"] = n, None

    def _search_reset(self, st, prefix):
        fin, P = st["fin"], st["P"]
        st["seqs"].zero_()
        st["seqs"][:, :P] = torch.tensor(prefix, dtype=I32, device=self.device)
        st["scores"].zero_()
        st["anc"].copy_(st["anc_init"])
        fin["count"].zero_(); fin["score"].fill_(-math.inf); fin["len"].zero_(); fin["active"].fill_(1)
        fin["n_active"].fill_(st["B"])
        st["step"].zero_()

    def _search_prepare(self, st, enc: Seq, enc_lens, prefix, len_penalty, unk_penalty, min_seq_len, use_graph, max_len,
                        banned=None, record=False, ngram=None):
        """(Re)initialise one cached search state in place for the sentences of `enc` and a length budget `max_len`
        (<= the state's allocated length); capture its graphs if needed."""
        c, M = self.cfg, self.M
        st["unk_penalty"] = float(unk_penalty)
        st["budget"].fill_(max_len)
        d = st["beam_desc"]
        if st.get("opts_cap") != (min_seq_len, float(len_penalty)) or st.get("unk_cap") != float(unk_penalty):
            d.min_len, d.len_penalty = min_seq_len, len_penalty
            st["opts_cap"] = (min_seq_len, float(len_penalty))  # compared as Python values: c_float rounds 0.9 and would recapture every call
            st["g_fwd"] = st["g_sel"] = st["g_sel_ban"] = st["g_sel_ngram"] = None  # scalar options are baked into the captured select graphs
            st["unk_cap"] = float(unk_penalty)
        st["ban_on"] = bool(banned)
        st["ngram_on"] = ngram or 0
        st["attn_on"] = record
        if record and st["attn_hist"] is None:
            st["attn_hist"] = torch.zeros((st["ML"], st["R"], st["S_enc"]), dtype=torch.float32, device=self.device)
            with self._state_lock:  # the cache budget now counts the history too
                self._evict_search_states(keep=st["key"])
        if banned:
            self._set_bans(st, banned)
        if ngram:
            self._set_ngram(st, ngram)
        if enc_lens is not None:
            st["enc_lens"].copy_(enc_lens)
        for i in range(c.dec_layers):
            self._lin(enc, f"text_decoder.layers.{i}.encoder_decoder_attn.kv", 2 * M, out=st["cross_kv"][i])
        self._search_reset(st, prefix)
        if use_graph and st["g_fwd"] is None:
            self._capture(st)
            self._search_reset(st, prefix)  # the warm-up touched position-0 cache rows and the search state
        if use_graph and banned and st["g_sel_ban"] is None:
            self._capture_ban(st)
            self._search_reset(st, prefix)
        if use_graph and ngram and st["g_sel_ngram"] is None:
            self._capture_ngram(st)
            self._search_reset(st, prefix)
        if use_graph and record and st["g_fwd_attn"] is None:
            self._capture_attn(st)
            self._search_reset(st, prefix)

    def _search_step(self, st, use_graph, select=True):
        ban, ngram, rec = st["ban_on"], st["ngram_on"], st["attn_on"]
        if use_graph:
            sel = "_ban" if ban else "_ngram" if ngram else ""
            st["g_fwd_attn" if rec else "g_fwd"].replay()
            if select:
                st["g_sel" + sel].replay()
            with self._count_lock:
                self.graph_kernels += (st["n_fwd_attn"] if rec else st["n_fwd"]) + (st["n_sel" + sel] if select else 0)
        else:
            self._decoder_step_forward(st, record=rec)
            if select:
                self._decoder_step_select(st, ban=ban, ngram=ngram)

    def _search_bootstrap_step(self, st, prefix, i, use_graph):
        """fairseq2.cpp:1162-1247: feed prefix[i], score prefix[i+1] (the top-K kernel reports the lprob of its
        `eos_idx` argument, here the next prefix token)."""
        lib, c = _lib.load(), self.cfg
        self._search_step(st, use_graph, select=False)
        self._topk(st, prefix[i + 1], 0.0)
        st["scores"][:, i + 1] = st["scores"][:, i] + st["eos_lprob"]
        check(lib.sb_step_advance(st["step"].data_ptr(), ops._stream()), "sb_step_advance")

    def _search_collect(self, st):
        fin, B = st["fin"], st["B"]
        cnt = fin["count"].cpu().tolist()
        scr = fin["score"].cpu().tolist()
        ln_ = fin["len"].cpu().tolist()
        sq = fin["seqs"].cpu()
        results, best = [], []
        for bi in range(B):
            hyps = [(scr[bi][j], sq[bi, j, :ln_[bi][j]].tolist()) for j in range(cnt[bi])]
            order = sorted(range(len(hyps)), key=lambda j: -hyps[j][0])
            results.append([hyps[j] for j in order])
            best.append(order[0] if order else -1)
        st["best_fin"] = best
        return results

    @torch.inference_mode()
    def beam_search(self, enc: Seq, enc_lens, prefix: List[int], beam=5, soft_max=(1, 200), hard_max=1024,
                    len_penalty=1.0, unk_penalty=0.0, min_seq_len=1, use_graph=True, cross_kv=None, state_len=None,
                    banned=None, record_attention=False, ngram=None):
        """Device-resident beam search.  Returns per sentence the finished hypotheses [(score, ids)], best first
        (semantics: fairseq2.cpp:1371-1608; see decode.cu).  `cross_kv` is ignored (kept for API stability): the
        static cross-attention K/V of the cached search state are recomputed from `enc`.
        `state_len`: allocate (and cache) the search state for this many positions instead of the length budget
        min(hard_max, a*S_enc + b); the budget is then a device scalar of the state, so searches whose budgets differ
        share one state and its captured graphs.  None: the state is sized by the budget.
        `banned`: token-id sequences of fairseq2's BannedSequenceProcessor, applied at every selecting step (not in the
        prefix bootstrap): a row whose last n-1 tokens equal a sequence's first n-1 cannot take its last token.
        `record_attention`: every step also keeps the last decoder layer's head-summed cross-attention weights, for
        `token_timestamps` (one more kernel per step, on a third captured graph of the state).
        `ngram`: the n-gram size of fairseq2's NGramRepeatBlockProcessor, applied where `banned` is: at every selecting
        step a row cannot take a token that would repeat one of its n-grams (the prompt's included).  Not combined with
        `banned`."""
        if ngram is not None:
            if isinstance(ngram, bool) or int(ngram) != ngram or ngram < 1:
                raise ValueError(f"the n-gram size must be an integer >= 1, got {ngram!r}")
            if banned:
                raise NotImplementedError("banned sequences and n-gram blocking cannot be combined in one search")
            ngram = int(ngram)
        if banned is not None:
            banned = [[int(t) for t in (x.tolist() if isinstance(x, torch.Tensor) else x)] for x in banned]
            V = self.cfg.text_vocab
            for x in banned:
                if not x:
                    raise ValueError("a banned sequence must not be empty")
                if not all(0 <= t < V for t in x):
                    raise ValueError(f"banned token ids must lie in [0, {V})")
        B, S_enc = enc.B, enc.T
        a, b = soft_max
        ML = hard_max if a <= 0 else min(hard_max, int(a * S_enc) + b)  # fairseq2.cpp:1097-1105
        P = len(prefix)
        assert 1 <= P < ML
        if ML > self.cfg.max_seq_len:  # fairseq2's position encoder raises here; embed_kernel would read past the sinusoid table
            raise ValueError(f"The input sequence length must be less than or equal to the maximum sequence length "
                             f"({self.cfg.max_seq_len}), but is {ML} instead.")
        assert enc.PH == 0 and enc.Tp == enc.T, "encoder output must be a halo-free Seq"
        ML_state = ML if state_len is None else max(ML, int(state_len))
        st = self._search_state(B, S_enc, ML_state, beam, P, enc_lens is not None, use_graph)
        self._search_prepare(st, enc, enc_lens, prefix, len_penalty, unk_penalty, min_seq_len, use_graph, ML, banned,
                             bool(record_attention), ngram)
        n_steps = ML - 1 - (P - 1)
        for i in range(P - 1):
            self._search_bootstrap_step(st, prefix, i, use_graph)
        done = 0
        while done < n_steps:
            chunk = min(32, n_steps - done)
            for _ in range(chunk):
                self._search_step(st, use_graph)
            done += chunk
            if done < n_steps and int(st["fin"]["n_active"].item()) == 0:
                break
        results = self._search_collect(st)
        st["enc_ptr"] = enc.buf.data_ptr()
        self._last_search_state = st
        return results

    @torch.inference_mode()
    def harvest_decoder_states(self, lengths: List[int]) -> Optional[Seq]:
        """Decoder output states of each sentence's best hypothesis, gathered from the per-step history of the last
        beam search (position t of a hypothesis lives in hist[t][slot_t]).  Same function of the same tokens as the
        reference's teacher-forced re-run of the decoder over the winning sequence minus its final EOS
        (inference/generator.py:281-299), without the second pass.  `lengths[b]` = len(hypothesis) - 1."""
        st = self._last_search_state
        if st is None or any(j < 0 for j in st["best_fin"]):
            return None
        M, dev = self.M, self.device
        B, L = len(lengths), max(lengths)
        t_idx = torch.arange(L, device=dev)[None, :]
        Bs = st["B"]
        sel = torch.tensor(st["best_fin"], dtype=torch.int64, device=dev)
        slots = st["fin"]["anc"][torch.arange(Bs, device=dev), sel][:, :L].to(torch.int64)  # (Bs, L)
        out = st["hist"][t_idx.expand(Bs, L), slots]                                         # (Bs, L, M) row gather
        lens = torch.tensor(lengths, dtype=I32, device=dev)
        out = out * (t_idx < lens[:, None].to(torch.int64))[:, :, None].to(out.dtype)             # zero the padding rows
        return Seq(B, L, M, lens=lens, buf=out.reshape(B * L, M).contiguous())

    def _best_hypotheses(self, st):
        """(index into the batch, winner index >= 0, generated-token count n excluding the EOS) of the last search."""
        best = st["best_fin"]
        sel = torch.tensor([max(j, 0) for j in best], dtype=torch.int64, device=self.device)
        lens = st["fin"]["len"][torch.arange(st["B"], device=self.device), sel].tolist()
        n = [ln - st["P"] - 1 if j >= 0 else 0 for ln, j in zip(lens, best)]
        return sel, n

    def _recorded_state(self):
        st = self._last_search_state
        if st is None or not st["attn_on"]:
            raise RuntimeError("the last beam_search of this thread did not run with record_attention=True")
        return st

    @torch.inference_mode()
    def harvest_attention(self) -> Tuple[torch.Tensor, List[int]]:
        """The recorded cross-attention rows of each sentence's best hypothesis: (B, max n, S_enc) fp32 on the device, row k
        of sentence b being decoder position P-1+k (the step that chose generated token k), zeros past n; and the
        generated-token counts n (EOS excluded).  Gathered along the winner's cache slots (fin_anc)."""
        st = self._recorded_state()
        sel, n = self._best_hypotheses(st)
        B, P, dev = st["B"], st["P"], self.device
        L = max(max(n), 1)
        slots = st["fin"]["anc"][torch.arange(B, device=dev), sel][:, P - 1:P - 1 + L].to(torch.int64)
        pos = torch.arange(P - 1, P - 1 + L, device=dev)[None, :].expand(B, L)
        out = st["attn_hist"][pos, slots]
        keep = torch.arange(L, device=dev)[None, :] < torch.tensor(n, device=dev)[:, None]
        return out * keep[:, :, None].to(out.dtype), n

    @torch.inference_mode()
    def token_timestamps(self, filter_width: int = 3) -> List[Tuple[List[int], List[float]]]:
        """Per sentence of the last (recording) beam search: the start bin of every generated token of its best hypothesis
        (sb_token_timestamps: inference/transcriber.py's _extract_timestamps on the device, over F = len - 2 encoder
        frames) and its per-token scores float32(cum[P+k] - cum[P+k-1]) of the hypothesis' cumulative scores."""
        st = self._recorded_state()
        sel, n = self._best_hypotheses(st)
        B, P, dev = st["B"], st["P"], self.device
        ar = torch.arange(B, device=dev)
        slots = st["fin"]["anc"][ar, sel].contiguous()
        starts = ops.token_timestamps(st["attn_hist"], slots, torch.tensor(n, dtype=I32, device=dev), st["enc_lens"], P,
                                      filter_width).cpu()
        cum = st["fin"]["scores"][ar, sel].cpu()
        out = []
        for b in range(B):
            c = cum[b, P - 1:P + n[b]]
            out.append((starts[b, :n[b]].tolist(), (c[1:] - c[:-1]).tolist()))
        return out

    # ------------------------------------------------------------------------------------------ a10 teacher-forced pass
    @torch.inference_mode()
    def decode_full(self, text_seqs: torch.Tensor, text_lens: torch.Tensor, enc: Seq, enc_lens, cross_kv=None) -> Seq:
        """UnitYModel.decode without a state bag over (B, L) ids (generator.py:294-299)."""
        c, M, H = self.cfg, self.M, self.H
        B, L = text_seqs.shape
        if cross_kv is None:
            st = self._last_search_state
            cross_kv = st["cross_kv"] if (st is not None and st.get("enc_ptr") == enc.buf.data_ptr()) else self._cross_kv(enc)
        xb = ops.embed_seq(text_seqs.to(I32).contiguous(), self.w["text_embed"], self.pos, math.sqrt(M), M)
        x = Seq(B, L, M, lens=text_lens, buf=xb)
        for i in range(c.dec_layers):
            p = f"text_decoder.layers.{i}"
            x = self._mha_self(self._ln(x, p + ".self_attn_layer_norm"), p + ".self_attn", x, causal=True)
            h = self._ln(x, p + ".encoder_decoder_attn_layer_norm")
            q = self._lin(h, p + ".encoder_decoder_attn.q_proj", M)
            kv = cross_kv[i].buf
            att = Seq(B, L, M)
            ops.attention(q.buf, kv[:, :M], kv[:, M:], att.buf, B, H, L, enc.T, L, 0, enc.Tp, enc.PH, enc_lens)
            x = self._lin(att, p + ".encoder_decoder_attn.output_proj", M, res1=x)
            x = self._ffn(self._ln(x, p + ".ffn_layer_norm"), p + ".ffn", c.dec_ffn_dim, ACT_RELU, x)
        return self._ln(x, "text_decoder.layer_norm")

    # ------------------------------------------------------------------------------------------ a11-a14 NAR T2U
    @torch.inference_mode()
    def t2u_encode(self, x: Seq) -> Seq:
        """The T2U's pre-LN Transformer encoder over the text decoder states (UnitYNART2UModel.encode, model.py:404-412,
        and UnitYT2UModel.encode, :292-298), keys masked by x.lens."""
        c = self.cfg
        for i in range(c.t2u_enc_layers):
            p = f"t2u_model.encoder.layers.{i}"
            x = self._mha_self(self._ln(x, p + ".self_attn_layer_norm"), p + ".self_attn", x)
            x = self._ffn(self._ln(x, p + ".ffn_layer_norm"), p + ".ffn", c.t2u_ffn_dim, ACT_RELU, x)
        return self._ln(x, "t2u_model.encoder.layer_norm")

    @torch.inference_mode()
    def t2u(self, dec_out: Seq, text_seqs: torch.Tensor, duration_factor: float = 1.0,
            durations: Optional[torch.Tensor] = None):
        """UnitYNART2UModel.forward (model.py:379-402) + argmax/pad/UnitTokenDecoder (generator.py:338-353).
        Returns units (B,U) int64 (pad -> 1 after decoding), unit_lens (B,), aux dict."""
        lib = _lib.load()
        c, M, dev = self.cfg, self.M, self.device
        B, L = dec_out.B, dec_out.T
        stream = ops._stream()
        t2u_enc = self.t2u_encode(dec_out)
        # --- NARDecoderFrontend (nar_decoder_frontend.py:300-334)
        ts = text_seqs.to(I32).contiguous()
        max_c = (L - 2) * self.max_chars + 1 if L > 2 else 1
        char_lens = torch.empty((B, L), dtype=I32, device=dev)
        char_seqs = torch.empty((B, max_c), dtype=I32, device=dev)
        char_seq_lens = torch.empty((B,), dtype=I32, device=dev)
        check(lib.sb_text_to_chars(ts.data_ptr(), L, B, self.tok_len.data_ptr(), self.tok_flags.data_ptr(),
                                   self.tok_chars.data_ptr(), self.max_chars, c.text_pad, c.text_unk, c.text_eos,
                                   char_lens.data_ptr(), char_seqs.data_ptr(), max_c, char_seq_lens.data_ptr(), stream),
              "sb_text_to_chars")
        Cn = max(int(char_seq_lens.max().item()), 1)  # host sync #1 (the reference syncs here too: .item() at :231)
        if Cn > c.max_seq_len:  # fairseq2's position encoder raises here; the kernel would read past the sinusoid table
            raise ValueError(f"The input sequence length must be less than or equal to the maximum sequence length "
                             f"({c.max_seq_len}), but is {Cn} instead.")
        P = "t2u_model.decoder_frontend"
        y = Seq(B, Cn, M, halo=1, lens=char_seq_lens)
        check(lib.sb_upsample_add(t2u_enc.buf.data_ptr(), t2u_enc.Tp, t2u_enc.PH, L, char_lens.data_ptr(),
                                  y.buf.data_ptr(), y.Tp, y.PH, Cn, B, M, self.pos.data_ptr(), self.w["alpha_char"].data_ptr(),
                                  self.w["char_embed"].data_ptr(), char_seqs.data_ptr(), max_c, math.sqrt(M), None, stream),
              "sb_upsample_add")
        dp = P + ".variance_adaptor.duration_predictor"
        h1 = ops.gemm(y, self.w[dp + ".conv1.0.w"], c.var_hidden, self.w[dp + ".conv1.0.b"], taps=c.var_kernel, act=ACT_RELU)
        h1 = self._ln(h1, dp + ".ln1", mask=True)
        h2 = ops.gemm(h1, self.w[dp + ".conv2.0.w"], c.var_hidden, self.w[dp + ".conv2.0.b"], taps=c.var_kernel, act=ACT_RELU)
        h2 = self._ln(h2, dp + ".ln2", mask=True)
        dur = torch.empty((B, Cn), dtype=I32, device=dev)
        check(lib.sb_durations(h2.buf.data_ptr(), h2.Tp, h2.PH, self.w[dp + ".proj.w"].data_ptr(), self.dur_bias, c.var_hidden,
                               char_seq_lens.data_ptr(), B, Cn, float(duration_factor), dur.data_ptr(), stream), "sb_durations")
        if durations is not None:  # VarianceAdaptor.forward(durations=...) override (length_regulator.py:275-283)
            dur = durations.to(device=dev, dtype=I32).contiguous()
        unit_lens = dur.sum(dim=1).to(I32)
        U = max(int(unit_lens.max().item()), 1)  # host sync #2 (reference: length_regulator.py:30)
        if U > c.max_seq_len:
            raise ValueError(f"The input sequence length must be less than or equal to the maximum sequence length "
                             f"({c.max_seq_len}), but is {U} instead.")
        halo = (c.fft_kernel - 1) // 2
        z = Seq(B, U, M, halo=halo, lens=unit_lens)
        check(lib.sb_upsample_add(y.buf.data_ptr(), y.Tp, y.PH, Cn, dur.data_ptr(), z.buf.data_ptr(), z.Tp, z.PH, U, B, M,
                                  self.pos.data_ptr(), self.w["alpha"].data_ptr(), None, None, 0, 0.0, None, stream),
              "sb_upsample_add")
        # --- FeedForwardTransformer (fft_decoder.py:65-77, fft_decoder_layer.py:177-231)
        for i in range(c.t2u_dec_layers):
            p = f"t2u_model.decoder.layers.{i}"
            s = self._mha_self(z, p + ".self_attn", z)
            z1 = self._ln(s, p + ".self_attn_layer_norm", mask=True)
            c1 = ops.gemm(z1, self.w[p + ".conv1d.conv1.w"], c.fft_inner_dim, self.w[p + ".conv1d.conv1.b"], taps=c.fft_kernel,
                          act=ACT_RELU)
            s2 = ops.gemm(c1, self.w[p + ".conv1d.conv2.w"], M, self.w[p + ".conv1d.conv2.b"], taps=c.fft_kernel, res1=z1)
            z = self._ln(s2, p + ".conv1d_layer_norm", mask=True)
        z = self._ln(z, "t2u_model.decoder.layer_norm", mask=True)
        ldv = (c.unit_vocab + 7) // 8 * 8
        logits = Seq(B, U, c.unit_vocab, z.PH, z.Tp, z.lens, dtype=torch.float32,
                     buf=torch.empty((B * z.Tp, ldv), dtype=torch.float32, device=dev))
        ops.gemm(z, self.w["unit_embed"], c.unit_vocab, None, out=logits, out_f32=True, mask=False)
        units = torch.empty((B, U), dtype=I32, device=dev)
        check(lib.sb_unit_argmax(logits.buf.data_ptr(), ldv, z.Tp, z.PH, U, B, c.unit_vocab, unit_lens.data_ptr(), c.unit_pad,
                                 c.unit_eos, units.data_ptr(), stream), "sb_unit_argmax")
        aux = dict(t2u_enc=t2u_enc, char_lens=char_lens, char_seqs=char_seqs[:, :Cn], char_seq_lens=char_seq_lens, dur=dur,
                   fft_out=z, logits=logits)
        return units.to(torch.int64), unit_lens, aux


def conv_transpose_taps(cw: torch.Tensor, u: int, k: int) -> torch.Tensor:
    """ConvTranspose1d(stride u, kernel k, padding (k - u) // 2) weights (cin, cout, k) -> (u * cout, 3 * cin) weights
    of a zero-padded 3-tap conv at the input rate whose u * cout outputs per input frame are the u output frames of
    that frame, phase-major: output frame q * u + p = sum_t w[p, :, t, :] . x[q + t - 1], tap j = p + pad - (t - 1) * u
    of the transposed conv.  Only k - u even (u * T output frames) with every tap j in [0, k) reached by some (p, t),
    i.e. u <= k <= 3 u, has this form; anything else raises ValueError instead of dropping taps."""
    cin, cout = cw.shape[0], cw.shape[1]
    if cw.shape[2] != k or u < 1 or (k - u) % 2 or not u <= k <= 3 * u:
        raise ValueError(f"ConvTranspose1d(stride {u}, kernel {k}) with weights {tuple(cw.shape)} is not a 3-tap conv "
                         f"over the input frames (needs k - u even and u <= k <= 3u)")
    pad = (k - u) // 2
    wt = torch.zeros(u, cout, 3, cin, dtype=cw.dtype)
    for p in range(u):
        for t in range(3):
            j = p + pad - (t - 1) * u
            if 0 <= j < k:
                wt[p, :, t, :] = cw[:, :, j].t()
    return wt.reshape(u * cout, 3 * cin)


class VocoderEngine:
    """Code-HiFiGAN (models/vocoder/{vocoder,codehifigan,hifigan}.py) on sb_gemm."""

    HALO0 = 5  # unit-rate halo; scales with the upsampling so that stage 1 has the 25 rows k=11,d=5 needs

    DUR_PREDICTOR_KEYS = tuple("code_generator.dur_predictor." + n for n in (
        "conv1.0.weight", "conv1.0.bias", "ln1.weight", "ln1.bias", "conv2.0.weight", "conv2.0.bias", "ln2.weight",
        "ln2.bias", "proj.weight", "proj.bias"))

    def __init__(self, cfg: VocoderConfig, state_dict: Dict[str, torch.Tensor], device="cuda"):
        # the duration predictor is optional, as in the reference (codehifigan.py:45-47): all of its tensors or none
        missing = [k for k in self.DUR_PREDICTOR_KEYS if k not in state_dict]
        if 0 < len(missing) < len(self.DUR_PREDICTOR_KEYS):
            raise ValueError(f"incomplete vocoder duration predictor: missing {missing}")
        self.has_dur_predictor = not missing
        _lib.require_cuda()
        self.cfg, self.device = cfg, torch.device(device)
        self.fused_resblocks = os.environ.get("SB_FUSED_RESBLOCK", "1") != "0"  # 16/32-channel stages: resblock.cu
        self._pack(state_dict)

    def _pack(self, sd):
        dev, c = self.device, self.cfg
        P = "code_generator."
        w: Dict[str, torch.Tensor] = {}

        def folded(name):  # weight_norm: w = g * v / ||v|| per dim-0 slice (hifigan.py:198-205 remove_weight_norm)
            v, g = sd[P + name + ".weight_v"].float(), sd[P + name + ".weight_g"].float()
            return g * v / v.flatten(1).norm(dim=1).view(-1, 1, 1)

        def conv(name):
            cw = folded(name)  # (out, in, k)
            w[name + ".w"] = cw.permute(0, 2, 1).reshape(cw.shape[0], -1).to(dev, F16).contiguous()
            w[name + ".b"] = sd[P + name + ".bias"].to(dev, torch.float32).contiguous()

        for n in ("dict", "spkr", "lang"):
            w[n] = sd[P + n + ".weight"].to(dev, F16).contiguous()
        conv("conv_pre")
        ch = c.upsample_initial_channel
        for i, (u, k) in enumerate(zip(c.upsample_rates, c.upsample_kernel_sizes)):
            w[f"ups.{i}.w"] = conv_transpose_taps(folded(f"ups.{i}"), u, k).to(dev, F16).contiguous()
            w[f"ups.{i}.b"] = sd[P + f"ups.{i}.bias"].float().repeat(u).to(dev).contiguous()
            for j in range(len(c.resblock_kernel_sizes)):
                rb = i * len(c.resblock_kernel_sizes) + j
                for d in range(len(c.resblock_dilation_sizes[j])):
                    conv(f"resblocks.{rb}.convs1.{d}")
                    conv(f"resblocks.{rb}.convs2.{d}")
        cp = folded("conv_post")  # (1, C, 7)
        w["conv_post.w"] = cp.permute(0, 2, 1).reshape(-1).to(dev, F16).contiguous()
        self.conv_post_bias = float(sd[P + "conv_post.bias"][0])
        if self.has_dur_predictor:
            dp = "dur_predictor."
            H, K = c.var_pred_hidden, c.var_pred_kernel
            for name, cin in (("conv1.0", c.embedding_dim), ("conv2.0", H)):
                cw = sd[P + dp + name + ".weight"]
                if tuple(cw.shape) != (H, cin, K) or K % 2 == 0:
                    raise ValueError(f"{P}{dp}{name}.weight has shape {tuple(cw.shape)}, expected ({H}, {cin}, {K}) "
                                     f"with an odd kernel")
                w[dp + name + ".w"] = cw.permute(0, 2, 1).reshape(H, -1).to(dev, F16).contiguous()  # (out, k, in)
                w[dp + name + ".b"] = sd[P + dp + name + ".bias"].to(dev, torch.float32).contiguous()
            for name in ("ln1", "ln2"):
                w[dp + name + ".w"] = sd[P + dp + name + ".weight"].to(dev, torch.float32).contiguous()
                w[dp + name + ".b"] = sd[P + dp + name + ".bias"].to(dev, torch.float32).contiguous()
            w[dp + "proj.w"] = sd[P + dp + "proj.weight"].reshape(-1).to(dev, F16).contiguous()
            self.dur_bias = float(sd[P + dp + "proj.bias"][0])
        self.w = w

    @torch.inference_mode()
    def __call__(self, units: torch.Tensor, lang_idx: List[int], spkr_idx: List[int]) -> torch.Tensor:
        """units (B,U) int -> waveform (B,1,U*hop) fp32  (CodeGenerator.forward with dur_prediction=False)."""
        B, U = units.shape
        x0 = Seq(B, U, self.cfg.model_in_dim, halo=self.HALO0)
        self._embed(units, lang_idx, spkr_idx, x0)
        return self._generate(x0)

    @torch.inference_mode()
    def resynthesize(self, units: torch.Tensor, lang_idx: List[int], spkr_idx: List[int],
                     durations: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """CodeGenerator.forward with dur_prediction=True (codehifigan.py:75-101): the duration predictor runs on the unit
        embeddings, row b's [lang | dict | spkr] frames are repeated by their durations to T_b = sum(dur[b]) frames, and
        the generator runs on the ragged batch with every row masked to its own length.
        units (B,U) int -> (wav (B,1,hop*max_b T_b) fp32, zero past hop*T_b in row b; wav_lens (B,) int64 on the host,
        = hop*T_b; durations (B,U) int32 on the device).  `durations` (B,U) replaces the predicted ones (as
        VarianceAdaptor.forward(durations=...) does for the T2U)."""
        x0, lens, tot, dur = self._expand(units, lang_idx, spkr_idx, durations)
        B = units.shape[0]
        if B > 1 and B * x0.Tp * self._max_rate() > self.MAX_GEMM_ROWS:
            # too many frames for one pass: the halves are generated on their own (each row is masked to its own length,
            # so a row's samples do not depend on the rows it is batched with), with the durations already predicted
            h = B // 2
            parts = [self.resynthesize(units[r0:r1], lang_idx[r0:r1], spkr_idx[r0:r1], dur[r0:r1])[0]
                     for r0, r1 in ((0, h), (h, B))]
            wav = torch.zeros((B, 1, max(p.shape[-1] for p in parts)), dtype=torch.float32, device=self.device)
            wav[:h, :, :parts[0].shape[-1]] = parts[0]
            wav[h:, :, :parts[1].shape[-1]] = parts[1]
            return wav, tot.to(torch.int64) * self.cfg.hop, dur
        return self._generate(x0, lens), tot.to(torch.int64) * self.cfg.hop, dur

    # one sb_gemm call covers at most 65535 row tiles of 128 rows (the grid's y extent)
    MAX_GEMM_ROWS = 65535 * 128

    def _fused_stage(self, cout: int) -> bool:
        """The stage's ResBlocks run as fused kernels (resblock.cu) rather than conv by conv on sb_gemm."""
        c = self.cfg
        return self.fused_resblocks and cout in (16, 32) and all(
            len(dl) == 3 and rk % 2 == 1 and rk <= 11 and (rk - 1) // 2 * max(dl) <= 32
            for rk, dl in zip(c.resblock_kernel_sizes, c.resblock_dilation_sizes))

    def _max_rate(self) -> int:
        """Rows per unit-rate frame of the longest sb_gemm of _generate: the last upsampling GEMM's input when the last
        stage's ResBlocks are fused, else the full hop (its ResBlock convs run on sb_gemm at the output rate)."""
        c = self.cfg
        cout = c.upsample_initial_channel // 2 ** len(c.upsample_rates)
        return c.hop // c.upsample_rates[-1] if self._fused_stage(cout) else c.hop

    def _expand(self, units, lang_idx, spkr_idx, durations=None):
        """Duration predictor + HardUpsampling of resynthesize() -> (x0 Seq (B, max T_b, model_in_dim) with rows past
        T_b zero, lens (1+stages, B) int32 on the device, T_b (B,) on the host, durations (B,U) int32)."""
        if not self.has_dur_predictor:
            raise NotImplementedError("this vocoder was loaded without duration-predictor weights "
                                      "(code_generator.dur_predictor.*)")
        lib = _lib.load()
        c, dev, w = self.cfg, self.device, self.w
        B, U = units.shape
        stream = ops._stream()
        dp = "dur_predictor."
        xu = Seq(B, U, c.model_in_dim, halo=(c.var_pred_kernel - 1) // 2)
        self._embed(units, lang_idx, spkr_idx, xu)
        # VariancePredictor (length_regulator.py:172-218, padding_mask None) on the dict channels of xu, read in place
        lo = c.lang_embedding_dim
        xd = Seq(B, U, c.embedding_dim, xu.PH, xu.Tp, buf=xu.buf[:, lo:lo + c.embedding_dim])
        h1 = ops.gemm(xd, w[dp + "conv1.0.w"], c.var_pred_hidden, w[dp + "conv1.0.b"], taps=c.var_pred_kernel, act=ACT_RELU)
        h1 = ops.layernorm(h1, w[dp + "ln1.w"], w[dp + "ln1.b"])
        h2 = ops.gemm(h1, w[dp + "conv2.0.w"], c.var_pred_hidden, w[dp + "conv2.0.b"], taps=c.var_pred_kernel, act=ACT_RELU)
        h2 = ops.layernorm(h2, w[dp + "ln2.w"], w[dp + "ln2.b"])
        dur = torch.empty((B, U), dtype=I32, device=dev)
        check(lib.sb_durations(h2.buf.data_ptr(), h2.Tp, h2.PH, w[dp + "proj.w"].data_ptr(), self.dur_bias,
                               c.var_pred_hidden, None, B, U, 1.0, dur.data_ptr(), stream), "sb_durations")
        if durations is not None:
            if tuple(durations.shape) != (B, U):
                raise ValueError(f"durations must have shape {(B, U)}, got {tuple(durations.shape)}")
            dur = durations.to(device=dev, dtype=I32).contiguous()
        # the one host sync: the expanded length sizes every buffer below (the reference syncs here too, in
        # repeat_interleave); the per-row totals are summed on the host from the copied durations
        dur_h = dur.cpu()
        tot = dur_h.sum(dim=1)
        if int(dur_h.min()) < 0 or int(tot.min()) < 1:
            raise ValueError(f"durations must be >= 0 with at least one frame per row (row totals {tot.tolist()})")
        T = int(tot.max())
        # row lengths at unit rate and after each upsampling stage, uploaded in one copy
        scale, scales = 1, [1]
        for u in c.upsample_rates:
            scale *= u
            scales.append(scale)
        lens = (tot.to(torch.int64)[None, :] * torch.tensor(scales)[:, None]).to(I32).to(dev)
        x0 = Seq(B, T, c.model_in_dim, halo=self.HALO0, lens=lens[0])
        # HardUpsampling of [lang | dict | spkr]: rows past each row's total are written as zeros
        check(lib.sb_upsample_add(xu.buf.data_ptr(), xu.Tp, xu.PH, U, dur.data_ptr(), x0.buf.data_ptr(), x0.Tp, x0.PH, T,
                                  B, c.model_in_dim, None, None, None, None, 0, 0.0, None, stream), "sb_upsample_add")
        return x0, lens, tot, dur

    def _embed(self, units: torch.Tensor, lang_idx: List[int], spkr_idx: List[int], x0: Seq) -> None:
        """x0 data rows = [lang | dict[unit] | spkr] (codehifigan.py:98-100)."""
        lib = _lib.load()
        c, dev, w = self.cfg, self.device, self.w
        B, U = units.shape
        stream = ops._stream()
        # NOTE: every tensor whose data_ptr() is handed to a kernel must stay referenced until after the launch;
        # a temporary freed earlier can be re-issued by the caching allocator to the next allocation.
        units_i = units.to(I32).contiguous()
        if os.environ.get("SB_CHECK_UNITS", "1") != "0":
            # torch's embedding would assert on an id outside the table; the gather kernel would read out of bounds.
            # UnitTokenDecoder maps control / language symbols to negative ids or ids >= num_embeddings (unit_tokenizer.py:231-238)
            lo, hi = int(units_i.min().item()), int(units_i.max().item())
            if lo < 0 or hi >= c.num_embeddings:
                raise IndexError(f"unit id out of range for the vocoder's {c.num_embeddings}-entry table (min {lo}, max {hi})")
        lang_t = torch.tensor(lang_idx, dtype=I32, device=dev)
        spkr_t = torch.tensor(spkr_idx, dtype=I32, device=dev)
        check(lib.sb_vocoder_embed(units_i.data_ptr(), U, B, w["dict"].data_ptr(), c.embedding_dim,
                                   w["lang"].data_ptr(), c.lang_embedding_dim, lang_t.data_ptr(), w["spkr"].data_ptr(),
                                   c.spkr_embedding_dim, spkr_t.data_ptr(), x0.buf.data_ptr(), x0.Tp, x0.PH, stream),
              "sb_vocoder_embed")

    def _generate(self, x0: Seq, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Generator.forward (hifigan.py:180-196) on x0 -> (B,1,T*hop) fp32.  lens (1+stages, B) int32: row b's length
        at unit rate and after each upsampling stage; every conv sees the rows past it as zero padding, and they are 0
        in the waveform.  None: every row has x0.T frames."""
        lib = _lib.load()
        c, dev, w = self.cfg, self.device, self.w
        B = x0.B
        stream = ops._stream()
        ch = c.upsample_initial_channel
        act = ops.gemm(x0, w["conv_pre.w"], ch, w["conv_pre.b"], taps=7, act=ACT_LRELU, slope=0.1)  # lrelu fused for ups[0]
        # every buffer below is fully written by a masked sb_gemm except its outermost halo rows (zero="edges")
        nk = len(c.resblock_kernel_sizes)
        nstage = len(c.upsample_rates)
        for i, u in enumerate(c.upsample_rates):
            cout = ch // (2 ** (i + 1))
            # ConvTranspose1d as a 3-tap GEMM producing u*cout values per input frame == u output frames of cout
            T, PHn, Tp = act.T * u, act.PH * u, act.Tp * u
            last_slope = 0.01 if i == nstage - 1 else 0.1  # F.leaky_relu default slope before conv_post (hifigan.py:192)
            L = None if lens is None else lens[i + 1]
            nxt_act = Seq(B, T, cout, PHn, Tp, lens=L, zero="edges")
            fused = self._fused_stage(cout)
            # masked at the input rate: row b's T_b input frames give its u*T_b output frames
            up_raw = Seq(act.B, act.T, u * cout, act.PH, act.Tp, lens=act.lens, zero="edges")
            up_act = None if fused else Seq(act.B, act.T, u * cout, act.PH, act.Tp, lens=act.lens, zero="edges")
            ops.gemm(act, w[f"ups.{i}.w"], u * cout, w[f"ups.{i}.b"], taps=3, out=up_raw, out2=up_act, out2_slope=0.1)
            x_raw = Seq(B, T, cout, PHn, Tp, lens=L, buf=up_raw.buf.view(B * Tp, cout))
            if fused:
                # narrow stages: each ResBlock is one kernel that keeps its time tile in shared memory (resblock.cu)
                xs = None
                for j, (rk, dil) in enumerate(zip(c.resblock_kernel_sizes, c.resblock_dilation_sizes)):
                    rb = i * nk + j
                    lastblock = j == nk - 1
                    acc = Seq(B, T, cout, PHn, Tp, lens=L, zero="edges")
                    names = [f"resblocks.{rb}.convs1.{di}" for di in range(3)], [f"resblocks.{rb}.convs2.{di}" for di in range(3)]
                    ops.hifigan_resblock(x_raw, [w[n + ".w"] for n in names[0]], [w[n + ".b"] for n in names[0]],
                                         [w[n + ".w"] for n in names[1]], [w[n + ".b"] for n in names[1]], rk, list(dil),
                                         res2=xs, gamma=(1.0 / nk) if lastblock else 1.0, out=acc,
                                         out2=nxt_act if lastblock else None, out2_slope=last_slope)
                    xs = acc
                act = nxt_act
                continue
            x_act = Seq(B, T, cout, PHn, Tp, lens=L, buf=up_act.buf.view(B * Tp, cout))
            xs = None
            for j, (rk, dil) in enumerate(zip(c.resblock_kernel_sizes, c.resblock_dilation_sizes)):
                rb = i * nk + j
                y_raw, y_act = x_raw, x_act
                for di, d in enumerate(dil):
                    t1 = ops.gemm(y_act, w[f"resblocks.{rb}.convs1.{di}.w"], cout, w[f"resblocks.{rb}.convs1.{di}.b"], taps=rk,
                                  dil=d, act=ACT_LRELU, slope=0.1)
                    lastpair = di == len(dil) - 1
                    if not lastpair:
                        n_raw = Seq(B, T, cout, PHn, Tp, lens=L, zero="edges")
                        n_act = Seq(B, T, cout, PHn, Tp, lens=L, zero="edges")
                        ops.gemm(t1, w[f"resblocks.{rb}.convs2.{di}.w"], cout, w[f"resblocks.{rb}.convs2.{di}.b"], taps=rk,
                                 res1=y_raw, out=n_raw, out2=n_act, out2_slope=0.1)
                        y_raw, y_act = n_raw, n_act
                    else:
                        # xs (+)= resblock output; the last resblock also applies the 1/num_kernels mean and the
                        # leaky-relu that feeds the next stage (hifigan.py:186-192)
                        lastblock = j == nk - 1
                        acc = Seq(B, T, cout, PHn, Tp, lens=L, zero="edges")
                        ops.gemm(t1, w[f"resblocks.{rb}.convs2.{di}.w"], cout, w[f"resblocks.{rb}.convs2.{di}.b"], taps=rk,
                                 res1=y_raw, res2=xs, gamma=(1.0 / nk) if lastblock else 1.0, out=acc,
                                 out2=nxt_act if lastblock else None, out2_slope=last_slope)
                        xs = acc
            act = nxt_act
        Tw = act.T
        wav = torch.empty((B, Tw), dtype=torch.float32, device=dev)
        check(lib.sb_conv_post_tanh(act.buf.data_ptr(), act.Tp, act.PH, Tw, ops._p(act.lens), act.C, B,
                                    w["conv_post.w"].data_ptr(), self.conv_post_bias, 7, wav.data_ptr(), wav.stride(0),
                                    stream), "sb_conv_post_tanh")
        return wav.view(B, 1, Tw)
