"""Synthetic, seeded stand-ins for the assets the reference downloads.

The reference resolves checkpoints and SentencePiece models through URLs
(cards/seamlessM4T_v2_large.yaml:10-11, cards/vocoder_v2.yaml:10) which are
unreachable offline.  This module produces, deterministically from a seed:

  * a state_dict with the *reference's parameter names and tensor layouts*
    (the names `convert_unity_checkpoint` produces, models/unity/loader.py:179-389;
    vocoder names per models/vocoder/loader.py:24-36) - random-init weights of the
    named architecture;
  * an NLLB-layout text tokenizer and a char tokenizer (layout documented in
    ggml/ggml_convert.py:57-154: `<pad>,<unk>,<s>,</s>`, pieces, `__lang__` x N,
    three data-source control symbols);
  * 16 kHz waveforms (SURVEY.md 8d: noise + sinusoids).

Both the CUDA path and the CPU oracle consume exactly these objects, so parity
tests compare implementations, not assets.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from .config import AlignerConfig, UnitYConfig, VocoderConfig, Wav2Vec2EncoderConfig

SPACE = "▁"


def _round_fp16(t: torch.Tensor) -> torch.Tensor:
    """Weights live on the fp16 grid (the reference loads its checkpoint in fp16 on CUDA,
    cli/m4t/predict/predict.py:207-212); kept in fp32 storage so the oracle can use them directly."""
    return t.to(torch.float16).to(torch.float32)


class _Init:
    def __init__(self, seed: int):
        self.g = torch.Generator().manual_seed(seed)
        self.sd: Dict[str, torch.Tensor] = {}

    def normal(self, name, shape, std):
        self.sd[name] = _round_fp16(torch.randn(shape, generator=self.g) * std)
        return self.sd[name]

    def uniform(self, name, shape, a):
        self.sd[name] = _round_fp16((torch.rand(shape, generator=self.g) * 2 - 1) * a)
        return self.sd[name]

    def linear(self, prefix, out_f, in_f, bias=True, gain=1.0):
        a = gain * math.sqrt(6.0 / (in_f + out_f))
        self.uniform(prefix + ".weight", (out_f, in_f), a)
        if bias:
            self.normal(prefix + ".bias", (out_f,), 0.02)

    def conv(self, prefix, out_c, in_c, k, bias=True, gain=1.0):
        std = gain / math.sqrt(in_c * k)
        self.normal(prefix + ".weight", (out_c, in_c, k), std)
        if bias:
            self.normal(prefix + ".bias", (out_c,), 0.02)

    def ln(self, prefix, dim):
        self.sd[prefix + ".weight"] = _round_fp16(1.0 + 0.05 * torch.randn(dim, generator=self.g))
        self.sd[prefix + ".bias"] = _round_fp16(0.02 * torch.randn(dim, generator=self.g))

    def mha(self, prefix, dim):
        for p in ("q_proj", "k_proj", "v_proj", "output_proj"):
            self.linear(f"{prefix}.{p}", dim, dim)


def make_unity_state_dict(cfg: UnitYConfig, seed: int = 0, logit_scale: float = 4.0,
                          with_t2u: Optional[bool] = None, dur_gain: float = 0.02, dur_bias: float = 0.0,
                          embed_scale: float = 0.25, dec_gain: float = 1.0) -> Dict[str, torch.Tensor]:
    """Random-init UnitY2 parameters under the reference's state_dict names (SURVEY 8b).

    With cfg.encoder_variant == "v1" the Conformer layers carry the w2v-BERT v1 parameters instead of the Shaw table and
    the conv-module LayerNorm: `self_attn.sdpa.r_proj` (no bias), `u_bias` / `v_bias` (H, 64) and
    `conv.batch_norm.{weight,bias,running_mean,running_var}` with non-trivial running statistics.  Its T2U is the
    autoregressive one (t2u_builder.py:311-427): `t2u_model.encoder.*`, `t2u_model.decoder_frontend.embed`,
    `t2u_model.decoder.layers.*` with `encoder_decoder_attn`, `t2u_model.decoder.layer_norm` and `t2u_model.final_proj`
    tied to the embedding.  It is drawn after every other tensor, and only with with_t2u=True: the default (None) draws
    the T2U of v2 architectures only, so the v1 text-only state dicts stay what they were.
    The v2 draws, and so every v2 state dict, are unchanged."""
    I = _Init(seed)
    M = cfg.model_dim
    v1 = cfg.encoder_variant == "v1"
    if with_t2u is None:
        with_t2u = not v1
    fd = cfg.fbank_channels * cfg.fbank_stride
    I.ln("speech_encoder_frontend.post_extract_layer_norm", fd)
    I.linear("speech_encoder_frontend.model_dim_proj", M, fd)
    for i in range(cfg.enc_layers):
        p = f"speech_encoder.inner.layers.{i}"
        for f in ("ffn1", "ffn2"):
            I.ln(f"{p}.{f}_layer_norm", M)
            I.linear(f"{p}.{f}.inner_proj", cfg.enc_ffn_dim, M)
            I.linear(f"{p}.{f}.output_proj", M, cfg.enc_ffn_dim)
        I.ln(f"{p}.self_attn_layer_norm", M)
        I.mha(f"{p}.self_attn", M)
        if v1:
            I.linear(f"{p}.self_attn.sdpa.r_proj", M, M, bias=False)
            I.normal(f"{p}.self_attn.sdpa.u_bias", (cfg.num_heads, cfg.head_dim), 0.5)
            I.normal(f"{p}.self_attn.sdpa.v_bias", (cfg.num_heads, cfg.head_dim), 0.5)
        else:
            I.normal(f"{p}.self_attn.sdpa.rel_k_embed.weight", (cfg.shaw_left + cfg.shaw_right + 1, cfg.head_dim),
                     cfg.head_dim ** -0.5)
        I.ln(f"{p}.conv_layer_norm", M)
        I.conv(f"{p}.conv.pointwise_conv1", 2 * M, M, 1, bias=False)
        I.normal(f"{p}.conv.depthwise_conv.weight", (M, 1, cfg.dw_kernel), 1.0 / math.sqrt(cfg.dw_kernel))
        if v1:
            bn = f"{p}.conv.batch_norm"
            I.ln(bn, M)  # weight around 1, bias around 0
            I.normal(bn + ".running_mean", (M,), 0.2)
            I.sd[bn + ".running_var"] = _round_fp16(0.25 + 1.5 * torch.rand(M, generator=I.g))
        else:
            I.ln(f"{p}.conv.layer_norm", M)
        I.conv(f"{p}.conv.pointwise_conv2", M, M, 1, bias=False)
        I.ln(f"{p}.layer_norm", M)
    I.ln("speech_encoder.inner_layer_norm", M)
    I.linear("speech_encoder.proj1", 4 * M, M)
    I.linear("speech_encoder.proj2", M, 4 * M)
    p = "speech_encoder.adaptor_layers.0"
    I.ln(f"{p}.residual_layer_norm", M)
    I.conv(f"{p}.residual_conv", 2 * M, M, cfg.adaptor_kernel)
    I.ln(f"{p}.self_attn_layer_norm", M)
    I.conv(f"{p}.self_attn_conv", 2 * M, M, cfg.adaptor_kernel)
    I.mha(f"{p}.self_attn", M)
    I.ln(f"{p}.ffn_layer_norm", M)
    I.linear(f"{p}.ffn.inner_proj", cfg.enc_ffn_dim, M)
    I.linear(f"{p}.ffn.output_proj", M, cfg.enc_ffn_dim)
    I.ln("speech_encoder.layer_norm", M)

    # text decoder (NLLB dense): tied embedding / final_proj (builder.py:451)
    emb = I.normal("text_decoder_frontend.embed.weight", (cfg.text_vocab, M), embed_scale * M ** -0.5)
    emb[cfg.text_pad].zero_()
    I.sd["final_proj.weight"] = emb
    for i in range(cfg.dec_layers):
        p = f"text_decoder.layers.{i}"
        I.ln(f"{p}.self_attn_layer_norm", M)
        I.mha(f"{p}.self_attn", M)
        I.ln(f"{p}.encoder_decoder_attn_layer_norm", M)
        I.mha(f"{p}.encoder_decoder_attn", M)
        I.ln(f"{p}.ffn_layer_norm", M)
        I.linear(f"{p}.ffn.inner_proj", cfg.dec_ffn_dim, M, gain=dec_gain)
        I.linear(f"{p}.ffn.output_proj", M, cfg.dec_ffn_dim, gain=dec_gain)
    I.ln("text_decoder.layer_norm", M)
    # SURVEY 7 hard-part 1: peak the logits (std ~= logit_scale) through the final LayerNorm gain so that
    # top-1/top-2 margins are far above fp16 drift.  The tied embedding is drawn with a *small* std
    # (embed_scale * M^-1/2): with an untrained tied embedding a larger input embedding makes the decoder echo
    # its own input token (h keeps the e_tok direction), which would make every decode step identical.
    I.sd["text_decoder.layer_norm.weight"] = _round_fp16(
        I.sd["text_decoder.layer_norm.weight"] * (logit_scale / embed_scale))

    if with_t2u and v1:
        _draw_ar_t2u(I, cfg, logit_scale, embed_scale)
    elif with_t2u:
        for i in range(cfg.t2u_enc_layers):
            p = f"t2u_model.encoder.layers.{i}"
            I.ln(f"{p}.self_attn_layer_norm", M)
            I.mha(f"{p}.self_attn", M)
            I.ln(f"{p}.ffn_layer_norm", M)
            I.linear(f"{p}.ffn.inner_proj", cfg.t2u_ffn_dim, M)
            I.linear(f"{p}.ffn.output_proj", M, cfg.t2u_ffn_dim)
        I.ln("t2u_model.encoder.layer_norm", M)
        uemb = I.normal("t2u_model.decoder_frontend.embed.weight", (cfg.unit_vocab, M), embed_scale * M ** -0.5)
        # SURVEY 7 hard-part 2: keep argmax inside the unit range [4, num_units+4) so the
        # reference vocoder's 10000-row embedding is never indexed out of range.
        uemb[:4].zero_()
        uemb[cfg.num_units + 4:].zero_()
        I.sd["t2u_model.final_proj.weight"] = uemb
        cemb = I.normal("t2u_model.decoder_frontend.embed_char.weight", (cfg.char_vocab, M), M ** -0.5)
        cemb[cfg.char_pad].zero_()
        I.sd["t2u_model.decoder_frontend.pos_emb_alpha"] = torch.ones(1)
        I.sd["t2u_model.decoder_frontend.pos_emb_alpha_char"] = torch.ones(1)
        p = "t2u_model.decoder_frontend.variance_adaptor.duration_predictor"
        I.conv(f"{p}.conv1.0", cfg.var_hidden, M, cfg.var_kernel)
        I.ln(f"{p}.ln1", cfg.var_hidden)
        I.conv(f"{p}.conv2.0", cfg.var_hidden, cfg.var_hidden, cfg.var_kernel)
        I.ln(f"{p}.ln2", cfg.var_hidden)
        # dur_gain/dur_bias: with the defaults round(exp(x)-1) == 0 -> clamped to 1, i.e. one unit per character
        # (SURVEY 8d: U = #chars = 495 at the headline point); tests raise them to exercise durations > 1.
        I.linear(f"{p}.proj", 1, cfg.var_hidden, gain=dur_gain)
        I.sd[f"{p}.proj.bias"] = _round_fp16(torch.tensor([dur_bias]))
        for i in range(cfg.t2u_dec_layers):
            p = f"t2u_model.decoder.layers.{i}"
            I.mha(f"{p}.self_attn", M)
            I.ln(f"{p}.self_attn_layer_norm", M)
            I.conv(f"{p}.conv1d.conv1", cfg.fft_inner_dim, M, cfg.fft_kernel)
            I.conv(f"{p}.conv1d.conv2", M, cfg.fft_inner_dim, cfg.fft_kernel)
            I.ln(f"{p}.conv1d_layer_norm", M)
        I.ln("t2u_model.decoder.layer_norm", M)
        I.sd["t2u_model.decoder.layer_norm.weight"] = _round_fp16(
            I.sd["t2u_model.decoder.layer_norm.weight"] * (logit_scale / embed_scale))
    return I.sd


def _draw_ar_t2u(I: _Init, cfg: UnitYConfig, logit_scale: float, embed_scale: float) -> None:
    """The autoregressive T2U of seamlessM4T_large (t2u_builder.py:311-427), scaled like the text decoder: a small tied
    unit embedding and a final LayerNorm gain that peaks the logits."""
    M = cfg.model_dim
    for i in range(cfg.t2u_enc_layers):
        p = f"t2u_model.encoder.layers.{i}"
        I.ln(f"{p}.self_attn_layer_norm", M)
        I.mha(f"{p}.self_attn", M)
        I.ln(f"{p}.ffn_layer_norm", M)
        I.linear(f"{p}.ffn.inner_proj", cfg.t2u_ffn_dim, M)
        I.linear(f"{p}.ffn.output_proj", M, cfg.t2u_ffn_dim)
    I.ln("t2u_model.encoder.layer_norm", M)
    uemb = I.normal("t2u_model.decoder_frontend.embed.weight", (cfg.unit_vocab, M), embed_scale * M ** -0.5)
    # control symbols and the language symbols score 0: the search only emits units in [4, num_units + 4), which the
    # vocoder's table can hold, and EOS only at the forced last step
    uemb[:4].zero_()
    uemb[cfg.num_units + 4:].zero_()
    I.sd["t2u_model.final_proj.weight"] = uemb
    for i in range(cfg.t2u_dec_layers):
        p = f"t2u_model.decoder.layers.{i}"
        I.ln(f"{p}.self_attn_layer_norm", M)
        I.mha(f"{p}.self_attn", M)
        I.ln(f"{p}.encoder_decoder_attn_layer_norm", M)
        I.mha(f"{p}.encoder_decoder_attn", M)
        I.ln(f"{p}.ffn_layer_norm", M)
        I.linear(f"{p}.ffn.inner_proj", cfg.t2u_ffn_dim, M)
        I.linear(f"{p}.ffn.output_proj", M, cfg.t2u_ffn_dim)
    I.ln("t2u_model.decoder.layer_norm", M)
    I.sd["t2u_model.decoder.layer_norm.weight"] = _round_fp16(
        I.sd["t2u_model.decoder.layer_norm.weight"] * (logit_scale / embed_scale))


def make_vocoder_state_dict(cfg: VocoderConfig, seed: int = 1, dur_predictor: bool = False, dur_gain: float = 0.3,
                            dur_bias: float = 1.0) -> Dict[str, torch.Tensor]:
    """Random-init Code-HiFiGAN parameters, weight-norm parametrised (weight_g/weight_v) exactly as the
    reference checkpoint stores them (models/vocoder/hifigan.py:44-176; loader.py:24-36).
    weight_g is drawn around ||v|| (PyTorch's default is exactly ||v||) so folding g*v/||v|| is exercised.

    dur_predictor=True adds the duration predictor (codehifigan.py:45-47, a VariancePredictor), drawn from its own
    generator so that every other tensor is the same as without it.  With the default dur_gain / dur_bias the predicted
    log-durations l spread about 1.0 +- 0.4, so round(exp(l) - 1) runs from clamped 1s to 5 or more (mean about 2)."""
    I = _Init(seed)
    P = "code_generator"

    def wn_conv(name, out_c, in_c, k, gain=1.0, transposed=False, stride=1):
        # Conv1d weight (out,in,k); ConvTranspose1d weight (in,out,k); norm over dims (1,2) per dim-0 slice
        fan_in = in_c * k / stride
        shape = (in_c, out_c, k) if transposed else (out_c, in_c, k)
        v = torch.randn(shape, generator=I.g) * (gain / math.sqrt(fan_in))
        g = v.flatten(1).norm(dim=1).view(-1, 1, 1) * (1.0 + 0.1 * torch.randn(shape[0], 1, 1, generator=I.g))
        I.sd[f"{P}.{name}.weight_v"] = _round_fp16(v)
        I.sd[f"{P}.{name}.weight_g"] = _round_fp16(g)
        I.sd[f"{P}.{name}.bias"] = _round_fp16(0.02 * torch.randn(out_c, generator=I.g))

    I.normal(f"{P}.dict.weight", (cfg.num_embeddings, cfg.embedding_dim), 1.0)
    I.normal(f"{P}.spkr.weight", (cfg.num_spkrs, cfg.spkr_embedding_dim), 1.0)
    I.normal(f"{P}.lang.weight", (cfg.num_langs, cfg.lang_embedding_dim), 1.0)
    ch = cfg.upsample_initial_channel
    wn_conv("conv_pre", ch, cfg.model_in_dim, 7)
    for i, (u, k) in enumerate(zip(cfg.upsample_rates, cfg.upsample_kernel_sizes)):
        cin, cout = ch // (2 ** i), ch // (2 ** (i + 1))
        wn_conv(f"ups.{i}", cout, cin, k, gain=1.4, transposed=True, stride=u)
        for j, (rk, dil) in enumerate(zip(cfg.resblock_kernel_sizes, cfg.resblock_dilation_sizes)):
            rb = i * len(cfg.resblock_kernel_sizes) + j
            for d in range(len(dil)):
                wn_conv(f"resblocks.{rb}.convs1.{d}", cout, cout, rk, gain=1.2)
                wn_conv(f"resblocks.{rb}.convs2.{d}", cout, cout, rk, gain=0.6)
    wn_conv("conv_post", 1, ch // (2 ** len(cfg.upsample_rates)), 7, gain=0.25)
    if dur_predictor:
        D = _Init(seed + 1000)
        p = f"{P}.dur_predictor"
        D.conv(f"{p}.conv1.0", cfg.var_pred_hidden, cfg.embedding_dim, cfg.var_pred_kernel)
        D.ln(f"{p}.ln1", cfg.var_pred_hidden)
        D.conv(f"{p}.conv2.0", cfg.var_pred_hidden, cfg.var_pred_hidden, cfg.var_pred_kernel)
        D.ln(f"{p}.ln2", cfg.var_pred_hidden)
        D.linear(f"{p}.proj", 1, cfg.var_pred_hidden, gain=dur_gain)
        D.sd[f"{p}.proj.bias"] = _round_fp16(torch.tensor([dur_bias]))
        I.sd.update(D.sd)
    return I.sd


# ----------------------------------------------------------------------------------------------
# tokenizers
# ----------------------------------------------------------------------------------------------
class VocabularyInfo:
    """Shim of fairseq2.data.VocabularyInfo (fields used by tests/unit/models/unity/test_unity.py)."""

    def __init__(self, size, unk_idx, bos_idx, eos_idx, pad_idx):
        self.size, self.unk_idx, self.bos_idx, self.eos_idx, self.pad_idx = size, unk_idx, bos_idx, eos_idx, pad_idx


class _PieceModel:
    """Stand-in for fairseq2's SentencePieceModel: index_to_token / token_to_index
    (call sites: models/unity/nar_decoder_frontend.py:138,247)."""

    def __init__(self, pieces: List[str], unk_idx: int):
        self.pieces = pieces
        self.index = {p: i for i, p in enumerate(pieces)}
        self.unk_idx = unk_idx

    def index_to_token(self, idx: int) -> str:
        return self.pieces[idx]

    def token_to_index(self, tok: str) -> int:
        return self.index.get(tok, self.unk_idx)


def _piece_name(i: int, nletters: int = 4) -> str:
    s = []
    for _ in range(nletters):
        s.append(chr(ord("a") + i % 26))
        i //= 26
    return SPACE + "".join(reversed(s))


class _TextEncoder:
    def __init__(self, tok: "SyntheticNllbTokenizer", prefix: List[str], suffix: List[str], device):
        self.tok = tok
        self.device = device
        self._prefix = [tok.model.token_to_index(p) for p in prefix]
        self._suffix = [tok.model.token_to_index(s) for s in suffix]
        self.prefix_indices = torch.tensor(self._prefix, dtype=torch.int64, device=device) if prefix else None
        self.suffix_indices = torch.tensor(self._suffix, dtype=torch.int64, device=device) if suffix else None

    def __call__(self, text: str) -> torch.Tensor:
        ids = list(self._prefix)
        for w in text.strip().split():
            ids.append(self.tok.model.token_to_index(SPACE + w))
        ids += self._suffix
        return torch.tensor(ids, dtype=torch.int64, device=self.device)


class _TextDecoder:
    def __init__(self, tok: "SyntheticNllbTokenizer"):
        self.tok = tok

    def __call__(self, ids) -> str:
        out = []
        for i in (ids.tolist() if hasattr(ids, "tolist") else ids):
            if i in self.tok.control_ids:
                continue
            out.append(self.tok.model.index_to_token(int(i)))
        return "".join(out).replace(SPACE, " ").strip()


class SyntheticNllbTokenizer:
    """NLLB-layout tokenizer over a synthetic piece inventory.

    Layout (ggml/ggml_convert.py:57-154; SURVEY 7.0): ``<pad>=0 <unk>=1 <s>=2 </s>=3``, ordinary pieces,
    then ``__lang__`` x len(langs), then ``<MINED_DATA> <MMT_BT_DATA> <SMT_BT_DATA>``.  Ordinary pieces are
    mostly "▁"+4 letters; a few punctuation / no-space pieces exercise the char-length merge rules of
    nar_decoder_frontend.py:158-225."""

    def __init__(self, vocab_size: int, langs: Sequence[str], default_lang: str = "eng"):
        n_ctrl_tail = len(langs) + 3
        n_ord = vocab_size - 4 - n_ctrl_tail
        assert n_ord > 40
        specials = [",", ".", "?", "!", "-", "ab", "cd", "efg", SPACE, "1"]
        pieces = ["<pad>", "<unk>", "<s>", "</s>"] + specials
        pieces += [_piece_name(i) for i in range(n_ord - len(specials))]
        pieces += [f"__{l}__" for l in langs] + ["<MINED_DATA>", "<MMT_BT_DATA>", "<SMT_BT_DATA>"]
        assert len(pieces) == vocab_size
        self.model = _PieceModel(pieces, 1)
        self.vocab_info = VocabularyInfo(size=vocab_size, unk_idx=1, bos_idx=2, eos_idx=3, pad_idx=0)
        self.langs = set(langs)
        self.default_lang = default_lang
        self.control_ids = set([0, 2, 3]) | set(range(vocab_size - n_ctrl_tail, vocab_size))

    def lang_index(self, lang: str) -> int:
        return self.model.token_to_index(f"__{lang}__")

    def create_encoder(self, *, task=None, lang=None, mode=None, device=None, pin_memory=False):
        if task is not None and task != "translation":
            raise ValueError(f"`task` must be 'translation', but is '{task}' instead.")
        lang = lang or self.default_lang
        if lang not in self.langs:
            raise ValueError(f"`lang` must be a supported language, but is '{lang}' instead.")
        if mode is None or mode == "source":
            pre, suf = [f"__{lang}__"], ["</s>"]
        elif mode == "target":
            pre, suf = ["</s>", f"__{lang}__"], []
        else:
            raise ValueError(f"`mode` must be 'source' or 'target', but is '{mode}' instead.")
        return _TextEncoder(self, pre, suf, device)

    def create_decoder(self):
        return _TextDecoder(self)

    def create_raw_encoder(self, *, device=None):
        """Encoder without prefix or suffix tokens (fairseq2 `create_raw_encoder`, used by MinTox to encode banned words).
        A word encodes to its "▁"-piece, or to UNK when the inventory lacks it.  A leading "★" becomes a token of its own
        (UNK: the inventory has no such piece) followed by the rest of the word, so that encode("★" + w)[1:] is w's
        encoding, as MinTox expects of a SentencePiece model."""
        return _RawTextEncoder(self, device)


class _RawTextEncoder(_TextEncoder):
    def __init__(self, tok: "SyntheticNllbTokenizer", device):
        super().__init__(tok, [], [], device)

    def __call__(self, text: str) -> torch.Tensor:
        ids = []
        for w in text.strip().split():
            if w.startswith("\u2605") and len(w) > 1:
                ids.append(self.tok.vocab_info.unk_idx)
                w = w[1:]
            ids.append(self.tok.model.token_to_index(SPACE + w))
        return torch.tensor(ids, dtype=torch.int64, device=self.device)


def char_pieces(text: str, is_known=None) -> List[str]:
    """The pieces a character-level SentencePiece model (`model_type=char`, default `nmt_nfkc` normaliser) encodes `text`
    to: NFKC; tab, newline and carriage return become spaces and other control characters are dropped; leading and
    trailing spaces are removed and runs of spaces collapse to one; a dummy space is prepended; every space is "▁" and
    every character is one piece, except that a run of characters the model lacks (`is_known(piece)` false) is one
    (unknown) piece.  An empty (or all-space) text gives no pieces."""
    import unicodedata
    out = []
    for ch in unicodedata.normalize("NFKC", text):
        if ch in "\t\n\r" or unicodedata.category(ch) == "Zs":
            out.append(" ")
        elif unicodedata.category(ch) != "Cc":
            out.append(ch)
    norm = " ".join(w for w in "".join(out).split(" ") if w)
    pieces = [SPACE] + [SPACE if ch == " " else ch for ch in norm] if norm else []
    if is_known is None:
        return pieces
    out = []
    for p in pieces:
        if out and not is_known(p) and not is_known(out[-1]):
            out[-1] += p
        else:
            out.append(p)
    return out


class RawCharEncoder:
    """The character model's raw encoder (fairseq2 SentencePieceEncoder without prefix or suffix): one id per piece of
    `char_pieces`, the unk id for a run of characters the model lacks.  `encode_as_tokens` gives the pieces themselves.
    model: anything with `token_to_index(piece)` that returns `unk_idx` for a piece it does not hold."""

    def __init__(self, model, unk_idx: int, device=None):
        self.model, self.unk_idx, self.device = model, unk_idx, device

    def _known(self, piece: str) -> bool:
        return self.model.token_to_index(piece) != self.unk_idx

    def __call__(self, text: str) -> torch.Tensor:
        return torch.tensor([self.model.token_to_index(p) for p in char_pieces(text, self._known)], dtype=torch.int64,
                            device=self.device)

    def encode_as_tokens(self, text: str) -> List[str]:
        return char_pieces(text, self._known)


class SyntheticCharTokenizer:
    """Char-level piece model (reference: models/unity/char_tokenizer.py:30; vocab 10943 for v2)."""

    def __init__(self, vocab_size: int):
        chars = [SPACE] + [chr(ord("a") + i) for i in range(26)] + list(",.?!-1")
        pieces = ["<unk>", "<pad>", "<s>", "</s>"] + chars
        pieces += [f"<c{i}>" for i in range(vocab_size - len(pieces))]
        assert len(pieces) == vocab_size, (len(pieces), vocab_size)
        self.model = _PieceModel(pieces, 0)
        self.vocab_info = VocabularyInfo(size=vocab_size, unk_idx=0, bos_idx=2, eos_idx=3, pad_idx=1)



def make_tokenizers(cfg: UnitYConfig) -> Tuple[SyntheticNllbTokenizer, SyntheticCharTokenizer]:
    return SyntheticNllbTokenizer(cfg.text_vocab, cfg.langs), SyntheticCharTokenizer(cfg.char_vocab)


# ----------------------------------------------------------------------------------------------
# audio
# ----------------------------------------------------------------------------------------------
def make_waveforms(batch: int, num_samples: int = 160000, seed: int = 1234, sample_rate: int = 16000) -> torch.Tensor:
    """(batch, num_samples) fp32 in [-1,1]: noise + 3 sinusoids per utterance (SURVEY 8d)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(num_samples, dtype=torch.float32) / sample_rate
    out = torch.empty(batch, num_samples)
    for b in range(batch):
        x = 0.1 * torch.randn(num_samples, generator=g)
        for _ in range(3):
            f = 100.0 + 3900.0 * torch.rand((), generator=g)
            a = 0.05 + 0.15 * torch.rand((), generator=g)
            ph = 2 * math.pi * torch.rand((), generator=g)
            x = x + a * torch.sin(2 * math.pi * f * t + ph)
        out[b] = x.clamp_(-1.0, 1.0)
    return out


def make_monotonic_state_dict(cfg: UnitYConfig, seed: int = 2, logit_scale: float = 4.0, embed_scale: float = 0.25,
                              dec_gain: float = 4.0, energy_layers: int = 4, energy_bias: float = -0.5) -> Dict[str, torch.Tensor]:
    """Random-init SeamlessStreaming monotonic text decoder (reference models/monotonic_decoder/builder.py:88-103
    `dense_1b`): an NLLB decoder whose every layer carries a PChooseLayer (p_choose.py:48-148).  Parameter names follow
    the module tree of `MonotonicDecoderModel` (text_decoder_frontend / text_decoder / final_proj)."""
    base = make_unity_state_dict(cfg, seed=seed, logit_scale=logit_scale, with_t2u=False, embed_scale=embed_scale, dec_gain=dec_gain)
    sd = {k: v for k, v in base.items() if k.startswith(("text_decoder", "final_proj"))}
    I = _Init(seed + 1000)
    M = cfg.model_dim
    for i in range(cfg.dec_layers):
        p = f"text_decoder.layers.{i}.p_choose_layer"
        for br in ("q_energy_proj", "k_energy_proj"):
            for l in range(energy_layers):
                I.linear(f"{p}.{br}.layers.{2 * l}", M, M, gain=1.2)  # Linear at even indices, ReLU at odd ones; gain keeps p_choose inside (0,1)
        I.sd[f"{p}.energy_bias"] = torch.full((1,), energy_bias)
    sd.update(I.sd)
    return sd


def make_wav2vec2_state_dict(cfg: Wav2Vec2EncoderConfig, seed: int = 3) -> Dict[str, torch.Tensor]:
    """Random-init wav2vec2 encoder weights under fairseq2's names (the names `convert_wav2vec2_checkpoint` produces),
    with the other synthetic models' init scale; the positional conv keeps its weight-norm pair (weight_g, weight_v)."""
    I = _Init(seed)
    M, F = cfg.model_dim, cfg.feature_dim
    c_in = 1
    for i, (c, k, _) in enumerate(cfg.feature_extractor_layer_descs):
        p = f"encoder_frontend.feature_extractor.layers.{i}"
        I.conv(p + ".conv", c, c_in, k)
        I.ln(p + ".layer_norm", c)
        c_in = c
    I.ln("encoder_frontend.post_extract_layer_norm", F)
    I.linear("encoder_frontend.model_dim_proj", M, F)
    K, G = cfg.pos_conv_kernel_size, cfg.num_pos_conv_groups
    p = "encoder_frontend.pos_encoder.conv"
    I.normal(p + ".weight_v", (M, M // G, K), 1.0 / math.sqrt(M // G * K))
    v = I.sd[p + ".weight_v"].double()
    # weight_g starts at the norm of weight_v per tap (what weight_norm's init gives), scaled so the fold is not a no-op
    I.sd[p + ".weight_g"] = _round_fp16((v.pow(2).sum((0, 1)).sqrt() * (1.0 + 0.1 * torch.randn(K, generator=I.g).double()))
                                        .float().reshape(1, 1, K))
    I.normal(p + ".bias", (M,), 0.02)
    for i in range(cfg.num_encoder_layers):
        p = f"encoder.layers.{i}"
        I.ln(p + ".self_attn_layer_norm", M)
        for q in ("q_proj", "k_proj", "v_proj", "output_proj"):
            I.linear(f"{p}.self_attn.{q}", M, M)
        I.ln(p + ".ffn_layer_norm", M)
        I.linear(p + ".ffn.inner_proj", cfg.ffn_inner_dim, M)
        I.linear(p + ".ffn.output_proj", M, cfg.ffn_inner_dim)
    I.ln("encoder.layer_norm", M)
    return I.sd


def make_kmeans_centroids(num: int, dim: int, seed: int = 4, scale: float = 1.0) -> torch.Tensor:
    """(num, dim) fp32 centroids on the fp16 grid (the layout KmeansModel's `.npy` is transposed to, kmeans.py:17-19)."""
    g = torch.Generator().manual_seed(seed)
    return _round_fp16(torch.randn(num, dim, generator=g) * scale)


def make_aligner_state_dict(cfg: AlignerConfig, seed: int = 5, embed_std: float = 1.0) -> Dict[str, torch.Tensor]:
    """Random-init UnitY2 aligner parameters under the reference's names (models/aligner/model.py:25-144 module tree:
    alignment_frontend.embed_{text,unit}, alignment_encoder.{t,f}_conv.<Sequential index>) on the fp16 grid."""
    I = _Init(seed)
    M = cfg.model_dim
    I.normal("alignment_frontend.embed_text.weight", (cfg.text_vocab_size, M), embed_std)
    I.normal("alignment_frontend.embed_unit.weight", (cfg.unit_vocab_size, cfg.feat_dim), embed_std)
    # Sequential indices: Permute12, then (Conv1d, ReLU, Dropout) per k3 layer, then Conv1d(k1), Dropout, Permute12
    for i in range(cfg.num_text_layers):
        k = 3 if i < cfg.num_text_layers - 1 else 1
        I.conv(f"alignment_encoder.t_conv.{1 + 3 * i}", M, M, k)
    c_in = cfg.feat_dim
    for i in range(cfg.num_feat_layers):
        k = 3 if i < cfg.num_feat_layers - 1 else 1
        I.conv(f"alignment_encoder.f_conv.{1 + 3 * i}", M, c_in, k)
        c_in = M
    return I.sd
