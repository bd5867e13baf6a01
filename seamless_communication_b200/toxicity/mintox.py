"""MinTox: re-decode the rows whose translation added toxicity, with the added words banned from the text search
(behavioural mirror of reference toxicity/mintox.py, with the deviations DESIGN.md "MinTox" lists: flagged rows are
always re-decoded alone, the caller's options are not mutated, and the merged unit batch is returned)."""
from __future__ import annotations

import dataclasses
import logging
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from ..inference.generator import BannedSequenceProcessor, SequenceGeneratorOptions
from ..nn import SequenceData, get_seqs_and_padding_mask
from .etox_bad_word_checker import ETOXBadWordChecker

logger = logging.getLogger(__name__)


def _extract_bad_words_with_batch_indices(source_texts: Sequence[str], target_texts: Sequence[str], source_lang: str,
                                          target_lang: str, bad_word_checker: ETOXBadWordChecker) -> Tuple[List[str], List[int]]:
    """Every row's extracted words, concatenated in row order, and the indices of the rows that have any."""
    words: List[str] = []
    rows: List[int] = []
    for i, (src, tgt) in enumerate(zip(source_texts, target_texts)):
        found = bad_word_checker.extract_bad_words(str(src), str(tgt), source_lang, target_lang)
        if found:
            rows.append(i)
            words += found
    return words, rows


def _replace_with_new_text_output_in_batch(original_texts: List[str], indices_with_toxicity: List[int],
                                           new_texts: Sequence[str]) -> None:
    """original_texts[indices[j]] = new_texts[j], in place (indices ascending)."""
    for j, i in enumerate(sorted(indices_with_toxicity)):
        original_texts[i] = new_texts[j]


def _replace_with_new_unit_output_in_batch(unit_tokenizer, original_units: Tensor, indices_with_toxicity_tensor: Tensor,
                                           new_units: Tensor) -> Tensor:
    """The batch with rows `indices` replaced by `new_units`; the narrower of the two is first padded on the right with
    the unit pad id.  Returns the merged tensor (it is `original_units`, updated in place, unless that had to be padded)."""
    pad = unit_tokenizer.vocab_info.pad_idx or 1
    width = max(original_units.size(1), new_units.size(1))
    if original_units.size(1) < width:
        original_units = F.pad(original_units, (0, width - original_units.size(1)), value=pad)
    if new_units.size(1) < width:
        new_units = F.pad(new_units, (0, width - new_units.size(1)), value=pad)
    original_units[indices_with_toxicity_tensor.to(original_units.device)] = new_units.to(original_units)
    return original_units


def banned_sequence_processor(text_tokenizer, banned_words: Sequence[str], device=None) -> BannedSequenceProcessor:
    """Each distinct word as its raw token ids, and once more as it encodes after a symbol ("★" + word, first token
    dropped), so that the word is banned after punctuation as well."""
    enc = text_tokenizer.create_raw_encoder(device=device)
    words = list(dict.fromkeys(banned_words))
    return BannedSequenceProcessor([enc(w) for w in words] + [enc(f"★{w}")[1:] for w in words])


def mintox_pipeline(model, text_tokenizer, unit_tokenizer, device, src_lang: str, tgt_lang: str, model_input: SequenceData,
                    input_modality, output_modality, src_texts: Sequence[str], original_texts: List[str],
                    original_units: Optional[Tensor] = None, unit_generation_ngram_filtering: bool = False,
                    text_generation_opts: Optional[SequenceGeneratorOptions] = None,
                    unit_generation_opts: Optional[SequenceGeneratorOptions] = None,
                    bad_word_checker: Optional[ETOXBadWordChecker] = None, duration_factor: float = 1.0,
                    prosody_encoder_input=None) -> Tuple[List[str], Optional[Tensor], List[int]]:
    """Check every row with `bad_word_checker`; re-decode the flagged rows alone with their added words banned from the
    text search, and merge the new texts (and units, for speech output) into the batch.  Returns the texts, the units
    (None for text output) and the flagged row indices; with no row flagged the inputs come back unchanged and nothing
    runs on the device."""
    from ..inference.translator import Modality, Translator

    assert bad_word_checker is not None
    text_opts = text_generation_opts or SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200))
    unit_opts = unit_generation_opts or SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(25, 50))
    words, rows = _extract_bad_words_with_batch_indices(src_texts, original_texts, src_lang, tgt_lang, bad_word_checker)
    speech = output_modality == Modality.SPEECH
    if not rows:
        return original_texts, (original_units if speech else None), rows
    logger.info("TOX src_lang=%s tgt_lang=%s added_tox=%d", src_lang, tgt_lang, len(rows))
    text_opts = dataclasses.replace(text_opts, step_processor=banned_sequence_processor(text_tokenizer, words, device))
    idx = torch.tensor(rows, device=model_input["seqs"].device)
    sub = dict(model_input, seqs=model_input["seqs"].index_select(0, idx),
               seq_lens=model_input["seq_lens"].index_select(0, idx.to(model_input["seq_lens"].device)))
    seqs, padding_mask = get_seqs_and_padding_mask(sub)
    new_texts, new_units = Translator.get_prediction(
        model, text_tokenizer, unit_tokenizer, seqs, padding_mask, input_modality, output_modality, tgt_lang, text_opts,
        unit_opts, unit_generation_ngram_filtering=unit_generation_ngram_filtering, duration_factor=duration_factor,
        prosody_encoder_input=prosody_encoder_input)
    texts = list(original_texts)
    _replace_with_new_text_output_in_batch(texts, rows, new_texts)
    if not speech:
        return texts, None, rows
    assert original_units is not None and new_units is not None
    units = _replace_with_new_unit_output_in_batch(unit_tokenizer, original_units, idx, new_units)
    return texts, units, rows
