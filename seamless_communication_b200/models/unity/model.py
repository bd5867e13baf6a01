"""UnitY2 model facade with the reference's method surface (models/unity/model.py:28-193, :331-441) over the CUDA
engine.  Tensors cross this boundary exactly as in the reference: (N,S,*) features / int64 ids in, (N,S,M) fp16 out."""
from __future__ import annotations

from typing import Dict, Optional, Tuple

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

    def __init__(self, cfg, engine: UnitYEngine):
        self.config = cfg
        self.engine = engine
        self.model_dim = cfg.model_dim
        self.input_modality = "speech"
        self.target_vocab_info = synthetic.VocabularyInfo(cfg.text_vocab, cfg.text_unk, cfg.text_bos, cfg.text_eos, cfg.text_pad)
        self.text_encoder = None  # Translator(input_modality=SPEECH) skips it (translator.py:97-104)
        self.text_decoder = engine
        self.prosody_encoder_model = None
        self.t2u_model = None
        if engine.has_t2u:
            uv = synthetic.VocabularyInfo(cfg.unit_vocab, 3, 0, cfg.unit_eos, cfg.unit_pad)
            self.t2u_model = UnitYNART2UModel(engine, uv)

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
        if state_bag is not None:
            raise NotImplementedError("incremental decoding runs inside the device-resident beam search")
        B, S, M = encoder_output.shape
        enc = Seq(B, S, M, buf=encoder_output.contiguous().view(B * S, M))
        tl = _lens(padding_mask, seqs.device)
        out = self.engine.decode_full(seqs, tl, enc, _lens(encoder_padding_mask, seqs.device))
        return out.buf.view(out.B, out.T, out.C), padding_mask

    def project(self, decoder_output: Tensor, decoder_padding_mask: Optional[PaddingMask]) -> SequenceModelOutput:
        from ... import ops
        B, S, M = decoder_output.shape
        logits = ops.gemm_raw(decoder_output.contiguous().view(B * S, M), self.engine.w["text_embed"], self.config.text_vocab,
                              out_f32=True)
        return SequenceModelOutput(logits.view(B, S, -1), self.target_vocab_info)


def load_unity_model(name_or_arch: str, device="cuda", dtype=torch.float16, state_dict: Optional[Dict[str, Tensor]] = None,
                     tokenizers=None, with_t2u: bool = True, seed: int = 0, checkpoint=None, synthetic: bool = False,
                     **synth_kw) -> UnitYModel:
    """Resolves an asset-card name to its architecture (reference: models/unity/loader.py:395-402) and builds the engine.
    Weights come from, in this order:
      * `state_dict` - parameters in the reference's fairseq2 naming;
      * `checkpoint` - a path or a loaded {"model": ...} mapping in the ORIGINAL fairseq naming (or fairseq2 naming),
        converted by models/checkpoint.py (the reference's convert_unity_checkpoint, loader.py:27-389);
      * `synthetic=True` - seeded random-init weights of the named architecture (synthetic.make_unity_state_dict;
        `seed` and further keywords go there).  Checkpoint URLs are unreachable offline, so tests and benchmarks use this.
    Without any of them a RuntimeError is raised: the reference would download the card's checkpoint, and silently
    answering with random weights instead would return garbage translations."""
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
    if state_dict is None and checkpoint is not None:
        from ..checkpoint import convert_unity_checkpoint, load_checkpoint_file
        ck = load_checkpoint_file(checkpoint) if isinstance(checkpoint, str) else checkpoint
        ctok = tokenizers[1]
        pieces = [ctok.model.index_to_token(i) for i in range(ctok.model.vocabulary_size)]
        state_dict = convert_unity_checkpoint(ck, char_pieces=pieces, nllb_vocab=cfg.text_vocab)["model"]
    if state_dict is None:
        if not synthetic:
            raise RuntimeError(f"no weights for '{name_or_arch}': pass state_dict=..., checkpoint=... (fairseq or fairseq2 naming) "
                               "or synthetic=True for seeded random-init weights; checkpoints cannot be downloaded here")
        state_dict = synthetic_mod.make_unity_state_dict(cfg, seed=seed, with_t2u=with_t2u, **synth_kw)
    elif not with_t2u:
        state_dict = {k: v for k, v in state_dict.items() if not k.startswith("t2u_model.")}
    return UnitYModel(cfg, UnitYEngine(cfg, state_dict, tokenizers, device=device))
