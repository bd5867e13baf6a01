"""Audio (or units) and a transcript -> the number of 20 ms units aligned to each character (reference
models/aligner/alignment_extractor.py:29-141): the XLS-R `UnitExtractor` followed by the UnitY2 aligner.

Deviations from the reference: nothing is resampled (a WAV file that is not 16 kHz raises), `plot=True` raises
NotImplementedError (matplotlib is not a dependency; the durations are what the plot would show), and the computation
is fp16 storage with fp32 accumulation whatever `dtype` says (DESIGN.md section 12).
"""
from __future__ import annotations

from typing import Any, List, Mapping, Optional, Sequence, Tuple, Union

import torch
from torch import Tensor

from ..unit_extractor import UnitExtractor
from .model import load_unity2_alignment_model


class AlignmentExtractor:
    """aligner_model_name_or_card: "nar_t2u_aligner" or "tiny_aligner"; unit_extractor_model_name_or_card /
    unit_extractor_output_layer / unit_extractor_kmeans_model_uri: as for `UnitExtractor` (units come from encoder layer
    output_layer - 1, as in the reference); without a unit extractor only units can be aligned.
    Weights: aligner_state_dict / aligner_checkpoint / char_tokenizer reach `load_unity2_alignment_model`,
    unit_extractor_state_dict / unit_extractor_checkpoint / num_centroids reach `UnitExtractor`; synthetic=True gives
    seeded weights to both (and seeded centroids when no k-means file is given)."""

    def __init__(self, aligner_model_name_or_card: str, unit_extractor_model_name_or_card: Optional[str] = None,
                 unit_extractor_output_layer: Optional[int] = None, unit_extractor_kmeans_model_uri: Optional[str] = None,
                 device: Union[str, torch.device] = "cuda", dtype: torch.dtype = torch.float16, *,
                 aligner_state_dict: Optional[Mapping[str, Tensor]] = None,
                 aligner_checkpoint: Union[str, Mapping[str, Any], None] = None, char_tokenizer=None,
                 unit_extractor_state_dict: Optional[Mapping[str, Tensor]] = None,
                 unit_extractor_checkpoint: Union[str, Mapping[str, Any], None] = None, num_centroids: int = 10000,
                 synthetic: bool = False):
        self.device, self.dtype = torch.device(device), dtype
        self.unit_extractor: Optional[UnitExtractor] = None
        self.unit_extractor_output_layer = 0
        if unit_extractor_model_name_or_card is not None:
            if unit_extractor_output_layer is None:
                raise ValueError("unit_extractor_output_layer is required with a unit extractor")
            self.unit_extractor = UnitExtractor(unit_extractor_model_name_or_card, unit_extractor_kmeans_model_uri, self.device,
                                                dtype, state_dict=unit_extractor_state_dict,
                                                checkpoint=unit_extractor_checkpoint, synthetic=synthetic,
                                                num_centroids=num_centroids)
            self.unit_extractor._check_layer(unit_extractor_output_layer - 1)
            self.unit_extractor_output_layer = unit_extractor_output_layer
        self.alignment_model = load_unity2_alignment_model(aligner_model_name_or_card, self.device,
                                                           state_dict=aligner_state_dict, checkpoint=aligner_checkpoint,
                                                           synthetic=synthetic, char_tokenizer=char_tokenizer)

    def prepare_audio(self, audio: Union[str, Tensor]) -> Tensor:
        """A WAV path (16 kHz, any channel count) or a (T,) / (C, T) float tensor -> (T,) fp32, averaged over channels
        (alignment_extractor.py:73-88)."""
        if isinstance(audio, str):
            from ...evaluate import decode_wav
            wav = decode_wav(audio, all_channels=True)
            if wav is None:
                raise ValueError(f"{audio}: not a decodable PCM WAV file")
            audio = wav
        if audio.dim() > 1:
            if audio.dim() != 2 or audio.size(0) >= audio.size(1):
                raise ValueError(f"Expected [Channel,Time] shape, but Channel > Time (shape {tuple(audio.shape)})")
            audio = audio.float().mean(0)
        return audio.to(self.device, torch.float32)

    def extract_units(self, audio: Tensor) -> Tensor:
        if self.unit_extractor is None:
            raise ValueError("a unit extractor is required to get units from audio")
        return self.unit_extractor.predict(audio, self.unit_extractor_output_layer - 1)

    def _units(self, audio: Union[str, Tensor]) -> Tensor:
        if isinstance(audio, Tensor) and not torch.is_floating_point(audio):
            return audio.reshape(-1)  # units given as the audio argument
        return self.extract_units(self.prepare_audio(audio))

    def _tokenize(self, units: Tensor, text: str, add_trailing_silence: bool) -> Tuple[Tensor, Tensor, List[str]]:
        if units.numel() == 0:
            raise ValueError("no units to align")
        fe = self.alignment_model.alignment_frontend
        text_ids = fe.tokenize_text(text, add_trailing_silence=add_trailing_silence)
        if text_ids.numel() == 0:
            raise ValueError("empty text: nothing to align the units to")
        return fe.tokenize_unit(units.cpu()), text_ids, fe.tokenize_text_to_tokens(text, add_trailing_silence)

    @torch.inference_mode()
    def extract_alignment(self, audio: Union[str, Tensor], text: str, plot: bool = False,
                          add_trailing_silence: bool = False) -> Tuple[Tensor, Tensor, List[str]]:
        """-> durations (1, T_text) int64 (units per character), text ids (1, T_text), the character pieces.  An integer
        tensor as `audio` is taken as units."""
        if plot:
            raise NotImplementedError("plotting needs matplotlib, which is not a dependency; the durations are returned")
        unit_ids, text_ids, tokens = self._tokenize(self._units(audio), text, add_trailing_silence)
        _, durations = self.alignment_model(text_ids[None], unit_ids[None])
        return durations, text_ids[None].to(self.device), tokens

    @torch.inference_mode()
    def extract_alignment_batch(self, audios_or_units: Sequence[Union[str, Tensor]], texts: Sequence[str],
                                add_trailing_silence: bool = False) -> List[Tuple[Tensor, Tensor, List[str]]]:
        """extract_alignment for many rows: the audio rows go through one `UnitExtractor.predict_batch`, then every row
        through one aligner forward.  Row b's result equals extract_alignment(audios_or_units[b], texts[b]) bit for bit."""
        if len(audios_or_units) != len(texts) or not texts:
            raise ValueError(f"{len(audios_or_units)} inputs for {len(texts)} texts")
        units: List[Optional[Tensor]] = [None] * len(texts)
        waves = []
        for b, a in enumerate(audios_or_units):
            if isinstance(a, Tensor) and not torch.is_floating_point(a):
                units[b] = a.reshape(-1)
            else:
                waves.append((b, self.prepare_audio(a)))
        if waves:
            if self.unit_extractor is None:
                raise ValueError("a unit extractor is required to get units from audio")
            ns = [len(w) for _, w in waves]
            batch = torch.zeros(len(waves), max(ns), device=self.device)
            for r, (_, w) in enumerate(waves):
                batch[r, :len(w)] = w
            got = self.unit_extractor.predict_batch(batch, ns, self.unit_extractor_output_layer - 1)
            for (b, _), u in zip(waves, got):
                units[b] = u
        rows = [self._tokenize(u, t, add_trailing_silence) for u, t in zip(units, texts)]
        tl, ul = [len(r[1]) for r in rows], [len(r[0]) for r in rows]
        tids = torch.zeros(len(rows), max(tl), dtype=torch.int64)
        uids = torch.zeros(len(rows), max(ul), dtype=torch.int64)
        for b, (u, t, _) in enumerate(rows):
            tids[b, :len(t)], uids[b, :len(u)] = t, u
        _, durations = self.alignment_model.engine.forward(tids, uids, tl, ul)
        return [(durations[b:b + 1, :tl[b]], t[None].to(self.device), toks) for b, (_, t, toks) in enumerate(rows)]

    def detokenize_text(self, tokenized_text_ids: Tensor) -> str:
        return self.alignment_model.alignment_frontend.decode_text(tokenized_text_ids)
