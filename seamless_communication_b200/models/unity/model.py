"""UnitY2 model facade with the reference's method surface (models/unity/model.py:28-193, :264-441) over the CUDA
engine.  Tensors cross this boundary exactly as in the reference: (N,S,*) features / int64 ids in, (N,S,M) fp16 out."""
from __future__ import annotations

import dataclasses
import threading
from typing import Dict, List, Optional, Tuple

import torch
from torch import Tensor

from ... import config as cfgmod
from ... import synthetic
from ... import synthetic as synthetic_mod
from ...engine import UnitYEngine
from ...nn import PaddingMask, SequenceModelOutput
from ...ops import Seq

I32 = torch.int32


def _lens(mask: Optional[PaddingMask], device) -> Optional[Tensor]:
    return None if mask is None else mask.seq_lens.to(device=device, dtype=I32)


def _decode(engine: UnitYEngine, seqs: Tensor, padding_mask: Optional[PaddingMask], encoder_output: Tensor,
            encoder_padding_mask: Optional[PaddingMask], state_bag) -> Tuple[Tensor, Optional[PaddingMask]]:
    """Teacher-forced decoder pass of an engine's NLLB-type decoder (no state bag)."""
    if state_bag is not None:
        raise NotImplementedError("incremental decoding runs inside the device-resident beam search")
    B, S, M = encoder_output.shape
    enc = Seq(B, S, M, buf=encoder_output.contiguous().view(B * S, M))
    out = engine.decode_full(seqs, _lens(padding_mask, seqs.device), enc, _lens(encoder_padding_mask, seqs.device))
    return out.buf.view(out.B, out.T, out.C), padding_mask


def _project(engine: UnitYEngine, decoder_output: Tensor, vocab_info) -> SequenceModelOutput:
    """Tied output projection of an engine's decoder: fp32 logits (N, S, V)."""
    from ... import ops
    B, S, M = decoder_output.shape
    logits = ops.gemm_raw(decoder_output.contiguous().view(B * S, M), engine.w["text_embed"], engine.cfg.text_vocab,
                          out_f32=True)
    return SequenceModelOutput(logits.view(B, S, -1), vocab_info)


# ---------------------------------------------------------------------------------------- autoregressive T2U (v1)
def t2u_decoder_config(cfg) -> "cfgmod.UnitYConfig":
    """The AR T2U decoder as the config of a decoder-only `UnitYEngine`: the same module type as the NLLB text decoder
    (t2u_builder.py:396-427, pre-LN, ReLU FFN; frontend :379-394 with _legacy_pad_idx = pad = 1, tied projection :323)
    with the T2U's layers, FFN width, unit vocabulary, special ids and position table."""
    return dataclasses.replace(cfg, name=cfg.name + "_t2u", dec_layers=cfg.t2u_dec_layers, dec_ffn_dim=cfg.t2u_ffn_dim,
                               text_vocab=cfg.unit_vocab, text_pad=cfg.unit_pad, text_unk=cfg.unit_unk,
                               text_bos=cfg.unit_bos, text_eos=cfg.unit_eos, max_seq_len=cfg.unit_max_seq_len)


_T2U_DEC_RENAMES = (("t2u_model.decoder_frontend.embed.weight", "text_decoder_frontend.embed.weight"),
                    ("t2u_model.final_proj.weight", "final_proj.weight"),
                    ("t2u_model.decoder.", "text_decoder."))


def t2u_decoder_state_dict(sd: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """The AR T2U decoder's parameters under the text decoder's names (`t2u_model.decoder.*` -> `text_decoder.*`, the
    unit embedding -> `text_decoder_frontend.embed.weight`, its tied projection -> `final_proj.weight`), which is what
    a decoder-only `UnitYEngine` and the oracle's decoder / beam search read.  Other keys are left out."""
    out: Dict[str, Tensor] = {}
    for k, v in sd.items():
        for src, dst in _T2U_DEC_RENAMES:
            if k.startswith(src):
                out[dst + k[len(src):]] = v
                break
    return out


class UnitYT2UModel:
    """models/unity/model.py:264-327: the autoregressive T2U of seamlessM4T_large.  `encode` runs the T2U encoder of
    the main engine; `decode` / `project` and the unit beam search run on `unit_engine`, a decoder-only `UnitYEngine`
    over the renamed decoder weights (its own search states, CUDA graphs and lanes: bind it in a LanePool next to the
    main engine)."""

    # the search state (KV caches, graphs) is cached per encoder length and allocated length; the T2U encoder output
    # is padded to a multiple of this many rows, with the true lengths masking the cross-attention, and the state is
    # allocated for the options' length ceiling, so text lengths share a few states
    S_ENC_BUCKET = 32

    def __init__(self, engine: UnitYEngine, unit_engine: UnitYEngine, vocab_info):
        self.engine, self.unit_engine = engine, unit_engine
        self.target_vocab_info = vocab_info
        self.model_dim = engine.M
        self._tls = threading.local()

    def encode(self, seqs: Tensor, padding_mask: Optional[PaddingMask]) -> Tuple[Tensor, Optional[PaddingMask]]:
        B, S, M = seqs.shape
        x = Seq(B, S, M, lens=_lens(padding_mask, seqs.device), buf=seqs.to(torch.float16).contiguous().view(B * S, M))
        out = self.engine.t2u_encode(x)
        return out.buf.view(B, S, M), padding_mask

    def decode(self, seqs: Tensor, padding_mask: Optional[PaddingMask], encoder_output: Tensor,
               encoder_padding_mask: Optional[PaddingMask], *, state_bag=None):
        return _decode(self.unit_engine, seqs, padding_mask, encoder_output, encoder_padding_mask, state_bag)

    def project(self, decoder_output: Tensor, decoder_padding_mask: Optional[PaddingMask]) -> SequenceModelOutput:
        return _project(self.unit_engine, decoder_output, self.target_vocab_info)

    def beam_search(self, enc: Seq, enc_lens: Optional[Tensor], prefix: List[int], beam=5, soft_max=(25, 50),
                    hard_max=1024, len_penalty=1.0, unk_penalty=0.0, bucket: bool = True, ngram: Optional[int] = None):
        """Unit beam search of BeamSearchSeq2SeqGenerator(echo_prompt=True) over the T2U encoder output `enc` (B, S, M)
        with per-row lengths `enc_lens` (int32 on the device; None: every row has S).  The length budget
        min(hard_max, a*S + b) uses the unpadded S, as the reference does.  With `bucket` (the results are the same):
          * the rows are padded to a multiple of S_ENC_BUCKET, masked through the lengths;
          * the search state is allocated for min(hard_max, unit_max_seq_len) positions (at least the budget), and the
            budget is applied on the device,
        so every text length of one bucket searches on one cached state with the same captured graphs.
        `ngram`: n-gram repeat blocking of that size (NGramRepeatBlockProcessor on the unit options; engine.beam_search)."""
        a, b = soft_max
        max_len = hard_max if a <= 0 else min(hard_max, int(a * enc.T) + b)
        state_len = None
        if bucket:
            state_len = max(max_len, min(hard_max, self.unit_engine.cfg.max_seq_len))
            if enc_lens is None:
                enc_lens = torch.full((enc.B,), enc.T, dtype=torch.int32, device=enc.buf.device)
            Sb = -(-enc.T // self.S_ENC_BUCKET) * self.S_ENC_BUCKET
            if Sb != enc.T:
                buf = torch.zeros((enc.B, Sb, enc.C), dtype=enc.buf.dtype, device=enc.buf.device)
                buf[:, :enc.T] = enc.buf.view(enc.B, enc.T, enc.C)
                enc = Seq(enc.B, Sb, enc.C, buf=buf.view(enc.B * Sb, enc.C))
                # held until this thread's next search: the engine recognises a thread's last encoder output by address
                # (decode_full reuses that search's cross-attention K/V), so the address must not go to another tensor
                self._tls.padded_enc = buf
        return self.unit_engine.beam_search(enc, enc_lens, prefix, beam=beam, soft_max=(0, 0), hard_max=max_len,
                                            len_penalty=len_penalty, unk_penalty=unk_penalty, state_len=state_len, ngram=ngram)


class UnitYNART2UModel:
    """models/unity/model.py:331-441."""

    def __init__(self, engine: UnitYEngine, vocab_info):
        self.engine = engine
        self.target_vocab_info = vocab_info

    def forward(self, text_decoder_output: Tensor, text_decoder_padding_mask: Optional[PaddingMask], text_seqs: Optional[Tensor],
                duration_factor: float = 1.0, film_cond_emb: Optional[Tensor] = None):
        if film_cond_emb is not None:
            raise NotImplementedError("FiLM conditioning (expressivity archs) is outside the S2ST hot path")
        B, L, M = text_decoder_output.shape
        dec = Seq(B, L, M, lens=_lens(text_decoder_padding_mask, text_decoder_output.device),
                  buf=text_decoder_output.contiguous().view(B * L, M))
        units, unit_lens, aux = self.engine.t2u(dec, text_seqs, duration_factor)
        self.last_units = units
        mask = PaddingMask(unit_lens.to(torch.int64), units.shape[1])
        # logits are kept in sequence layout on device; expose the dense (B,U,V) view the reference returns
        lg = aux["logits"]
        logits = lg.buf.view(lg.B, lg.Tp, -1)[:, lg.PH:lg.PH + lg.T, :self.target_vocab_info.size]
        return SequenceModelOutput(logits, self.target_vocab_info), mask, aux["dur"]

    __call__ = forward


class UnitYModel:
    """models/unity/model.py:28-193."""

    def __init__(self, cfg, engine: UnitYEngine, unit_engine: Optional[UnitYEngine] = None):
        self.config = cfg
        self.engine = engine
        self.model_dim = cfg.model_dim
        self.input_modality = "speech"
        self.target_vocab_info = synthetic.VocabularyInfo(cfg.text_vocab, cfg.text_unk, cfg.text_bos, cfg.text_eos, cfg.text_pad)
        self.text_encoder = None  # Translator(input_modality=SPEECH) skips it (translator.py:97-104)
        self.text_decoder = engine
        self.prosody_encoder_model = None
        self.t2u_model = None
        uv = synthetic.VocabularyInfo(cfg.unit_vocab, cfg.unit_unk, cfg.unit_bos, cfg.unit_eos, cfg.unit_pad)
        if engine.has_t2u:
            self.t2u_model = UnitYNART2UModel(engine, uv)
        elif unit_engine is not None:
            self.t2u_model = UnitYT2UModel(engine, unit_engine, uv)

    def eval(self):
        return self

    def encode(self, seqs: Tensor, padding_mask: Optional[PaddingMask]):
        if self.input_modality == "speech":
            return self.encode_speech(seqs, padding_mask)
        if self.input_modality == "text":
            return self.encode_text(seqs, padding_mask)
        raise RuntimeError(f"`input_modality` must be 'speech' or 'text', but is '{self.input_modality}' instead.")

    def encode_speech(self, seqs: Tensor, padding_mask: Optional[PaddingMask]):
        out, lens = self.engine.encode_speech(seqs.to(torch.float16).contiguous(), _lens(padding_mask, seqs.device))
        self._last_enc = out
        mask = None if lens is None else PaddingMask(lens.to(torch.int64), out.T)
        return out.buf.view(out.B, out.T, out.C), mask

    def encode_text(self, seqs: Tensor, padding_mask: Optional[PaddingMask]):
        raise ValueError("`encode_text()` requires a text encoder, but the current UnitY model does not have one.")

    def decode(self, seqs: Tensor, padding_mask: Optional[PaddingMask], encoder_output: Tensor,
               encoder_padding_mask: Optional[PaddingMask], *, state_bag=None):
        return _decode(self.engine, seqs, padding_mask, encoder_output, encoder_padding_mask, state_bag)

    def project(self, decoder_output: Tensor, decoder_padding_mask: Optional[PaddingMask]) -> SequenceModelOutput:
        return _project(self.engine, decoder_output, self.target_vocab_info)

    @property
    def engines(self) -> List[UnitYEngine]:
        """Every engine holding search states (the main one, and the AR T2U's unit engine): what a LanePool binds."""
        t2u = self.t2u_model
        return [self.engine] + ([t2u.unit_engine] if isinstance(t2u, UnitYT2UModel) else [])


def _layer_count(sd: Dict[str, Tensor], prefix: str) -> Optional[int]:
    """1 + the largest layer index under `prefix` ("...layers."), or None when the state dict has no such layer."""
    idx = [int(k[len(prefix):].split(".", 1)[0]) for k in sd if k.startswith(prefix)]
    return max(idx) + 1 if idx else None


def check_state_dict(sd: Dict[str, Tensor], cfg) -> None:
    """Refuse weights of another architecture before anything is built: the layer counts of the speech encoder, the
    text decoder and the T2U encoder and decoder (each where the state dict has it), the text decoder's FFN width and the
    vocabulary size of its tied table must be the config's.  Raises ValueError naming the first mismatch."""
    checks = [("speech encoder layers", _layer_count(sd, "speech_encoder.inner.layers."), cfg.enc_layers),
              ("text decoder layers", _layer_count(sd, "text_decoder.layers."), cfg.dec_layers)]
    ffn = sd.get("text_decoder.layers.0.ffn.inner_proj.weight")
    checks.append(("text decoder FFN width", None if ffn is None else ffn.shape[0], cfg.dec_ffn_dim))
    emb = sd.get("final_proj.weight", sd.get("text_decoder_frontend.embed.weight"))
    checks.append(("text vocabulary size", None if emb is None else emb.shape[0], cfg.text_vocab))
    checks += [("T2U encoder layers", _layer_count(sd, "t2u_model.encoder.layers."), cfg.t2u_enc_layers),
               ("T2U decoder layers", _layer_count(sd, "t2u_model.decoder.layers."), cfg.t2u_dec_layers)]
    for what, got, want in checks:
        if got is not None and got != want:
            raise ValueError(f"the weights do not fit architecture '{cfg.name}': {what} {got}, the architecture has {want}")


def load_unity_model(name_or_arch: str, device="cuda", dtype=torch.float16, state_dict: Optional[Dict[str, Tensor]] = None,
                     tokenizers=None, with_t2u: bool = True, seed: int = 0, checkpoint=None, synthetic: bool = False,
                     decoder_weight_dtype=torch.float16, **synth_kw) -> UnitYModel:
    """Resolves an asset-card name to its architecture (reference: models/unity/loader.py:395-402) and builds the engine.
    Weights come from, in this order:
      * `state_dict` - parameters in the reference's fairseq2 naming;
      * `checkpoint` - a path or a loaded {"model": ...} mapping in the ORIGINAL fairseq naming (or fairseq2 naming),
        converted by models/checkpoint.py (the reference's convert_unity_checkpoint, loader.py:27-389);
      * `synthetic=True` - seeded random-init weights of the named architecture (synthetic.make_unity_state_dict;
        `seed` and further keywords go there).  Checkpoint URLs are unreachable offline, so tests and benchmarks use this.
    Without any of them a RuntimeError is raised: the reference would download the card's checkpoint, and silently
    answering with random weights instead would return garbage translations.

    A w2v-BERT v1 architecture (`seamlessM4T_large` -> "base") has an autoregressive T2U: it is built when the weights
    hold its unit projection (`t2u_model.final_proj.weight`, or `decoder.output_projection` in fairseq naming) and
    `with_t2u` is set; otherwise the model runs speech-to-text only.  The text encoder is never built (text input is not
    supported) and its keys are dropped.

    The weights of `seamlessM4T_medium` are checked against the architecture first (`check_state_dict`): layer counts,
    the decoder's FFN width and the vocabulary size.  A mismatch raises ValueError.

    `decoder_weight_dtype=torch.float8_e4m3fn` runs the text decoder's beam search (and the AR T2U's unit search) on
    weight-only FP8: its six products per layer and the tied projection read e4m3 weights with one power-of-two scale
    per output feature.  The model computed is exactly the fp16 model on `dequantize_decoder_weights(state_dict, cfg)`
    (models/fp8_weights.py).  The default, torch.float16, runs the weights as given."""
    arch = cfgmod.MODEL_CARDS.get(name_or_arch, name_or_arch)
    if arch not in cfgmod.UNITY_ARCHS:
        raise ValueError(f"unknown model card / architecture '{name_or_arch}'")
    if dtype != torch.float16:
        raise ValueError("the sm_90a kernels compute in fp16 with fp32 accumulation; pass dtype=torch.float16")
    cfg = cfgmod.UNITY_ARCHS[arch]()
    if tokenizers is None:
        if not synthetic:
            raise RuntimeError("no tokenizers given: pass tokenizers=(text_tokenizer, char_tokenizer) matching the weights "
                               "(the SentencePiece models of the asset card are not reachable offline), or synthetic=True")
        tokenizers = synthetic_mod.make_tokenizers(cfg)
    v1 = cfg.encoder_variant == "v1"
    if state_dict is None and checkpoint is not None:
        from ..checkpoint import convert_unity_checkpoint, load_checkpoint_file
        ck = load_checkpoint_file(checkpoint) if isinstance(checkpoint, str) else checkpoint
        if v1:  # the text encoder (fairseq text_encoder.*) is not built; the AR T2U has no character table
            ck = {**ck, "model": {k: v for k, v in ck["model"].items() if not k.startswith("text_encoder.")}}
            pieces = None
        else:
            ctok = tokenizers[1]
            pieces = [ctok.model.index_to_token(i) for i in range(ctok.model.vocabulary_size)]
        state_dict = convert_unity_checkpoint(ck, char_pieces=pieces, nllb_vocab=cfg.text_vocab)["model"]
    if state_dict is None:
        if not synthetic:
            raise RuntimeError(f"no weights for '{name_or_arch}': pass state_dict=..., checkpoint=... (fairseq or fairseq2 naming) "
                               "or synthetic=True for seeded random-init weights; checkpoints cannot be downloaded here")
        state_dict = synthetic_mod.make_unity_state_dict(cfg, seed=seed, with_t2u=with_t2u, **synth_kw)
    elif not with_t2u or v1:
        drop = ("text_encoder.", "text_encoder_frontend.") if v1 else ()
        drop += () if with_t2u else ("t2u_model.",)
        state_dict = {k: v for k, v in state_dict.items() if not k.startswith(drop)}
    if arch == "medium":
        check_state_dict(state_dict, cfg)
    unit_engine = None
    if v1:
        ar = {k: v for k, v in state_dict.items() if k.startswith("t2u_model.")}
        state_dict = {k: v for k, v in state_dict.items() if k not in ar or k.startswith("t2u_model.encoder.")}
        if "t2u_model.final_proj.weight" in ar:
            unit_engine = UnitYEngine(t2u_decoder_config(cfg), t2u_decoder_state_dict(ar), (None, None), device=device,
                                      decoder_weight_dtype=decoder_weight_dtype)
        else:  # no AR T2U (an S2TT-only checkpoint): its encoder is not built either
            state_dict = {k: v for k, v in state_dict.items() if not k.startswith("t2u_model.")}
    return UnitYModel(cfg, UnitYEngine(cfg, state_dict, tokenizers, device=device, decoder_weight_dtype=decoder_weight_dtype),
                      unit_engine)
