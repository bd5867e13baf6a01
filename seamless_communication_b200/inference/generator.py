"""Text + unit generation for UnitY2 (behavioural mirror of reference inference/generator.py:39-364).

`SequenceGeneratorOptions` and `UnitYGenerator` keep the reference's names, arguments and error behaviour; the
work behind them is the device-resident beam search and the NAR T2U of `engine.py`."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, List, Optional, Tuple

import torch
from torch import Tensor

from ..models.unity import UnitTokenizer, UnitYModel, UnitYT2UModel
from ..nn import PaddingMask
from ..ops import Seq

I32 = torch.int32


def remove_consecutive_repeated_ngrams(sequence: List[int], min_size: int = 1, max_size: int = 40) -> List[int]:
    """Drops the first copy of every immediately repeated n-gram (generator.py:39-57)."""
    assert 1 <= min_size <= max_size
    drop = set()
    start = 0
    while start < len(sequence):
        for k in range(max_size, min_size - 1, -1):
            if sequence[start:start + k] == sequence[start + k:start + 2 * k]:
                drop |= set(range(start, start + k))
                start += k - 1
                break
        start += 1
    return [tok for i, tok in enumerate(sequence) if i not in drop]


def filter_unit_ngrams(units: Tensor) -> Tensor:
    """`ngram_filtering` of the AR T2U's decoded units (generator.py:356-362): batch 1 only, as in the reference."""
    if units.size(0) > 1:
        raise NotImplementedError("unit ngram_filtering is not implemented for batch_size > 1.")
    arr = remove_consecutive_repeated_ngrams(units[0].tolist())
    return torch.tensor(arr).to(units).unsqueeze(0)


@dataclass
class SequenceGeneratorOptions:
    """generator.py:59-84 (same fields and defaults)."""

    beam_size: int = 5
    soft_max_seq_len: Tuple[int, int] = (1, 200)
    hard_max_seq_len: int = 1024
    step_processor: Optional[Any] = None
    unk_penalty: float = 0.0
    len_penalty: float = 1.0


@dataclass
class TextGenOutput:
    hypotheses: List[List[Tuple[float, List[int]]]]
    encoder_output: Tensor
    encoder_padding_mask: Optional[PaddingMask]


class UnitYGenerator:
    """generator.py:87-364.  Cheap to construct (the reference rebuilds it on every get_prediction call)."""

    def __init__(self, model: UnitYModel, text_tokenizer, target_lang: str, unit_tokenizer: Optional[UnitTokenizer] = None,
                 text_opts: Optional[SequenceGeneratorOptions] = None, unit_opts: Optional[SequenceGeneratorOptions] = None) -> None:
        model.eval()
        self.model = model
        self.text_opts = text_opts or SequenceGeneratorOptions()
        # generator.py:205-210: the AR T2U's own default (speech sequences are much longer than text)
        self.unit_opts = unit_opts or SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=5000)
        if model.text_decoder is None:
            raise ValueError("`UnitYGenerator` requires a text decoder, but the current UnitY model does not have one.")
        if self.text_opts.step_processor is not None:
            raise NotImplementedError("step processors (MinTox banned sequences) are outside the S2ST hot path")
        self.text_tokenizer = text_tokenizer
        enc = text_tokenizer.create_encoder(task="translation", lang=target_lang, mode="target")
        self.prefix = enc.prefix_indices.tolist()  # [</s>, __lang__]
        self.text_decoder = text_tokenizer.create_decoder()
        self.unit_decoder = None
        self.unit_prefix_indices = None
        self.reuse_decoder_states = True  # False: recompute them with the teacher-forced pass, as the reference does
        if unit_tokenizer is not None:
            if model.t2u_model is None:
                raise ValueError("`model` does not have a T2U sub-model when `unit_tokenizer` is not None.")
            self.unit_decoder = unit_tokenizer.create_decoder()
            self.unit_prefix_indices = unit_tokenizer.create_encoder(lang=target_lang).prefix_indices
            if isinstance(model.t2u_model, UnitYT2UModel) and self.unit_opts.step_processor is not None:
                raise NotImplementedError("step processors (MinTox banned sequences) are outside the S2ST hot path")

    @torch.inference_mode()
    def __call__(self, source_seqs: Tensor, source_padding_mask: Optional[PaddingMask], input_modality: str = "speech",
                 output_modality: str = "speech", ngram_filtering: bool = False, duration_factor: float = 1.0,
                 prosody_encoder_input=None) -> Tuple[List[str], Optional[Tensor]]:
        if input_modality == "speech":
            enc_out, enc_mask = self.model.encode_speech(source_seqs, source_padding_mask)
        elif input_modality == "text":
            if self.model.text_encoder is None:
                raise ValueError("Please set `use_text_encoder` to `True` in your model config to encode text.")
            enc_out, enc_mask = self.model.encode_text(source_seqs, source_padding_mask)
        else:
            raise ValueError(f"Unsupported input_modality: {input_modality}")
        eng = self.model.engine
        B, S, M = enc_out.shape
        enc = Seq(B, S, M, buf=enc_out.view(B * S, M))
        enc_lens = None if enc_mask is None else enc_mask.seq_lens.to(device=enc_out.device, dtype=I32)
        o = self.text_opts
        hyps = eng.beam_search(enc, enc_lens, self.prefix, beam=o.beam_size, soft_max=o.soft_max_seq_len,
                               hard_max=o.hard_max_seq_len, len_penalty=o.len_penalty, unk_penalty=o.unk_penalty)
        for h in hyps:
            if not h:
                raise RuntimeError("The sequence generator returned no hypothesis at index 0. Please file a bug report.")
        text_seq_list = [h[0][1] for h in hyps]
        texts = [self.text_decoder(s) for s in text_seq_list]
        self.last_text_output = TextGenOutput(hyps, enc_out, enc_mask)
        if output_modality == "text":
            return texts, None

        pad = self.model.target_vocab_info.pad_idx
        L = max(len(s) for s in text_seq_list)
        text_seqs = torch.full((B, L), pad, dtype=torch.int64)
        for i, s in enumerate(text_seq_list):
            text_seqs[i, :len(s)] = torch.tensor(s)
        text_seqs = text_seqs[:, :-1].contiguous().to(enc_out.device)  # "trim the final EOS" (generator.py:287)
        text_lens = torch.tensor([len(s) - 1 for s in text_seq_list], dtype=I32, device=enc_out.device)
        # generator.py:294-299 re-runs the decoder teacher-forced over the winning sequences; the same states were
        # already computed during the search and are gathered from its history instead (engine.harvest_decoder_states)
        dec = eng.harvest_decoder_states([len(s) - 1 for s in text_seq_list]) if self.reuse_decoder_states else None
        if dec is None:
            dec = eng.decode_full(text_seqs, text_lens, enc, enc_lens)
        assert self.model.t2u_model is not None and self.unit_decoder is not None
        if isinstance(self.model.t2u_model, UnitYT2UModel):
            return texts, self._generate_units_ar(dec, text_lens, ngram_filtering)
        units, unit_lens, aux = eng.t2u(dec, text_seqs, duration_factor)
        # engine.t2u already applied argmax -> pad mask -> UnitTokenDecoder (generator.py:346-353) on device
        self.last_unit_output = dict(unit_lens=unit_lens, text_seqs=text_seqs, dec_out=dec, **aux)
        return texts, units

    def _generate_units_ar(self, dec: Seq, text_lens: Tensor, ngram_filtering: bool) -> Tensor:
        """generator.py:316-362 for the AR T2U: T2U encoder over the decoder states (text padding mask), unit beam search
        from the prefix [eos, lang] (echo_prompt=True: the hypotheses hold it), best hypothesis per row padded with the
        pad symbol, UnitTokenDecoder.  `last_unit_output["unit_lens"]` holds each row's decoded length (its EOS, turned
        into the pad symbol, included)."""
        t2u = self.model.t2u_model
        t2u_enc = self.model.engine.t2u_encode(dec)
        o = self.unit_opts
        hyps = t2u.beam_search(t2u_enc, text_lens, self.unit_prefix_indices.tolist(), beam=o.beam_size,
                               soft_max=o.soft_max_seq_len, hard_max=o.hard_max_seq_len, len_penalty=o.len_penalty,
                               unk_penalty=o.unk_penalty)
        for h in hyps:
            if not h:
                raise RuntimeError("The sequence generator returned no hypothesis at index 0. Please file a bug report.")
        seqs = [h[0][1] for h in hyps]
        unit_seqs = torch.full((len(seqs), max(len(s) for s in seqs)), t2u.target_vocab_info.pad_idx, dtype=torch.int64)
        for i, s in enumerate(seqs):
            unit_seqs[i, :len(s)] = torch.tensor(s)
        units = self.unit_decoder(unit_seqs)
        if ngram_filtering:
            units = filter_unit_ngrams(units)
        self.last_unit_output = dict(hypotheses=hyps, t2u_enc=t2u_enc, dec_out=dec,
                                     unit_lens=[units.size(1)] if ngram_filtering else [len(s) - 1 for s in seqs])
        return units
