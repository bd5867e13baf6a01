"""`Translator`: the drop-in boundary of the S2ST hot path (behavioural mirror of reference
inference/translator.py:53-428): same constructor / predict / get_prediction signatures, same enums, same errors."""
from __future__ import annotations

from dataclasses import dataclass
from enum import Enum, auto
from typing import List, Optional, Tuple, Union, cast

import threading

import torch
from torch import Tensor

from .. import config as cfgmod
from .. import ops
from ..models.unity import UnitTokenizer, UnitYModel, UnitYT2UModel, load_unity_model
from ..models.vocoder import Vocoder, load_vocoder_model
from ..nn import PaddingMask, SequenceData, get_seqs_and_padding_mask
from .generator import SequenceGeneratorOptions, UnitYGenerator


class Task(Enum):
    S2ST = auto()
    S2TT = auto()
    T2ST = auto()
    T2TT = auto()
    ASR = auto()


class Modality(Enum):
    SPEECH = "speech"
    TEXT = "text"


@dataclass
class BatchedSpeechOutput:
    units: List[List[int]]
    audio_wavs: List[Tensor]
    sample_rate: int = 16000


class Translator:
    _tls = threading.local()  # the calling thread's last generator (LanePool workers call predict concurrently)

    def __init__(self, model_name_or_card: Union[str, UnitYModel], vocoder_name_or_card: Union[str, Vocoder, None], device,
                 text_tokenizer=None, apply_mintox: bool = False, dtype=torch.float16,
                 input_modality: Optional[Modality] = None, output_modality: Optional[Modality] = None, **model_kw):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            # the reference silently switches to fp32 on CPU (translator.py:110-111); this implementation has no CPU path
            raise RuntimeError("seamless_communication_b200.Translator needs a CUDA device (sm_90a); no CPU fallback exists.")
        if apply_mintox:
            raise NotImplementedError("MinTox re-decoding is outside the S2ST hot path (SURVEY.md 2.1 P14)")
        with_t2u = output_modality != Modality.TEXT  # translator.py:105-107
        if isinstance(model_name_or_card, UnitYModel):
            self.model = model_name_or_card
        else:
            if text_tokenizer is not None and "tokenizers" not in model_kw:
                # the engine's T2U character tables and the prefix ids are built from ITS tokenizer pair: a different decode-side
                # tokenizer would silently produce wrong units (reference: one tokenizer object serves both, translator.py:118-127)
                raise ValueError("pass tokenizers=(text_tokenizer, char_tokenizer) so that the engine is built with the same "
                                 "tokenizer, or build the UnitYModel yourself")
            self.model = load_unity_model(model_name_or_card, device=self.device, dtype=dtype, with_t2u=with_t2u, **model_kw)
        self.model.eval()
        self.dtype = dtype
        if text_tokenizer is not None and text_tokenizer is not self.model.engine.text_tokenizer:
            raise ValueError("text_tokenizer differs from the tokenizer the model's engine was built with")
        self.text_tokenizer = self.model.engine.text_tokenizer
        self.unit_tokenizer: Optional[UnitTokenizer] = None
        if self.model.t2u_model is not None:
            c = self.model.config
            arch = "nar_multilingual_v2" if c.name.endswith("v2") else c.name
            self.unit_tokenizer = UnitTokenizer(c.num_units, list(c.unit_langs), arch)
        self.apply_mintox = apply_mintox
        self.vocoder: Optional[Vocoder] = None
        if vocoder_name_or_card is not None and output_modality != Modality.TEXT:
            self.vocoder = vocoder_name_or_card if isinstance(vocoder_name_or_card, Vocoder) else \
                load_vocoder_model(vocoder_name_or_card, device=self.device, dtype=dtype, synthetic=bool(model_kw.get("synthetic", False)))
            self.vocoder.eval()

    # -- fbank + collate (translator.py:135-146): both run on device here ---------------------------------------
    def convert_to_fbank(self, decoded_audio: dict) -> dict:
        wav = decoded_audio["waveform"]  # (T, C) channel-last, as the reference's AudioDecoder returns it
        if wav.dim() == 2:
            wav = wav[:, 0]
        wav = wav.to(self.device, torch.float32).contiguous()
        n = wav.numel()
        frames = 0 if n < 400 else 1 + (n - 400) // 160
        fb, _ = ops.fbank(wav.view(1, -1), torch.tensor([n], dtype=torch.int32, device=self.device), max(frames, 1))
        return {**decoded_audio, "fbank": fb[0, :frames]}

    def collate(self, item) -> dict:
        fb = item["fbank"] if isinstance(item, dict) else item
        T = fb.shape[0]
        Tp = T + (T % 2)  # pad_to_multiple=2
        out = torch.zeros((1, Tp, fb.shape[1]), dtype=fb.dtype, device=fb.device)
        out[0, :T] = fb
        return {"fbank": {"seqs": out, "seq_lens": torch.tensor([T], device=fb.device), "is_ragged": Tp != T}}

    def fbank_batch(self, waves: Tensor, num_samples: Optional[Tensor] = None) -> SequenceData:
        """Batched device frontend: (N, T) fp32 waveforms -> SequenceData of standardised fbank (N, frames, 80)."""
        waves = waves.to(self.device, torch.float32).contiguous()
        N, T = waves.shape
        ns = torch.full((N,), T, dtype=torch.int32, device=self.device) if num_samples is None else \
            num_samples.to(self.device, torch.int32)
        max_frames = 0 if T < 400 else 1 + (T - 400) // 160
        ld = max_frames + (max_frames % 2)
        fb, frames = ops.fbank(waves, ns, max(ld, 2))
        return {"seqs": fb, "seq_lens": frames, "is_ragged": num_samples is not None}

    @classmethod
    def get_prediction(cls, model: UnitYModel, text_tokenizer, unit_tokenizer: Optional[UnitTokenizer], seqs: Tensor,
                       padding_mask: Optional[PaddingMask], input_modality: Modality, output_modality: Modality, tgt_lang: str,
                       text_generation_opts: SequenceGeneratorOptions, unit_generation_opts: Optional[SequenceGeneratorOptions],
                       unit_generation_ngram_filtering: bool = False, duration_factor: float = 1.0,
                       prosody_encoder_input=None) -> Tuple[List[str], Optional[Tensor]]:
        generator = UnitYGenerator(model, text_tokenizer, tgt_lang, unit_tokenizer if output_modality == Modality.SPEECH else None,
                                   text_opts=text_generation_opts, unit_opts=unit_generation_opts)
        cls._last_generator = cls._tls.generator = generator
        return generator(seqs, padding_mask, input_modality.value, output_modality.value,
                         ngram_filtering=unit_generation_ngram_filtering, duration_factor=duration_factor,
                         prosody_encoder_input=prosody_encoder_input)

    @staticmethod
    def get_modalities_from_task_str(task_str: str) -> Tuple[Modality, Modality]:
        try:
            task = Task[task_str.upper()]
        except KeyError:
            raise ValueError(f"Unsupported task: {task_str}")
        if task == Task.S2ST:
            return Modality.SPEECH, Modality.SPEECH
        if task in (Task.S2TT, Task.ASR):
            return Modality.SPEECH, Modality.TEXT
        if task == Task.T2TT:
            return Modality.TEXT, Modality.TEXT
        return Modality.TEXT, Modality.SPEECH

    @torch.inference_mode()
    def predict(self, input: Union[str, Tensor, SequenceData], task_str: str, tgt_lang: str, src_lang: Optional[str] = None,
                text_generation_opts: Optional[SequenceGeneratorOptions] = None,
                unit_generation_opts: Optional[SequenceGeneratorOptions] = None, spkr: Optional[int] = -1,
                sample_rate: int = 16000, unit_generation_ngram_filtering: bool = False, duration_factor: float = 1.0,
                prosody_encoder_input=None, src_text=None) -> Tuple[List[str], Optional[BatchedSpeechOutput]]:
        input_modality, output_modality = self.get_modalities_from_task_str(task_str)
        if output_modality == Modality.SPEECH and self.model.config.encoder_variant == "v1":
            if self.model.t2u_model is None:
                raise NotImplementedError(f"{task_str.upper()} on {self.model.config.name} needs its autoregressive T2U (the "
                                          "v1 AR T2U model), which this model was loaded without; S2TT and ASR run")
            if input_modality == Modality.TEXT:
                raise NotImplementedError(f"{task_str.upper()} on {self.model.config.name} needs text input (the NLLB text "
                                          "encoder), which is not implemented; S2ST, S2TT and ASR are")
        if self.apply_mintox and not (src_lang is not None or src_text is not None):
            raise ValueError("`src_lang` must be specified when `apply_mintox` is `True` or you need to specify src_text.")
        if isinstance(input, dict):
            src = cast(SequenceData, input)
        elif input_modality == Modality.SPEECH:
            audio = input
            if isinstance(audio, str):
                raise NotImplementedError("audio file decoding (libsndfile) is outside the hot path; pass a waveform tensor")
            assert audio.dim() <= 2, "The audio tensor can't be more than 2 dimensions."
            if audio.dim() == 1:
                audio = audio.unsqueeze(1)
            elif audio.dim() == 2 and audio.size(0) < audio.size(1):
                audio = audio.transpose(0, 1)  # (bsz, seq_len) -> (seq_len, bsz), as the reference does
            decoded_audio = {"waveform": audio, "sample_rate": sample_rate, "format": -1}
            src = self.collate(self.convert_to_fbank(decoded_audio))["fbank"]
        else:
            if src_lang is None:
                raise ValueError("src_lang must be specified for T2ST, T2TT tasks.")
            raise NotImplementedError("text input needs the NLLB text encoder, which is outside the S2ST hot path")
        seqs, padding_mask = get_seqs_and_padding_mask(src)
        if text_generation_opts is None:
            text_generation_opts = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200))
        if unit_generation_opts is None:
            unit_generation_opts = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(25, 50))
        texts, units = self.get_prediction(self.model, self.text_tokenizer, self.unit_tokenizer, seqs, padding_mask,
                                           input_modality, output_modality, tgt_lang, text_generation_opts,
                                           unit_generation_opts, unit_generation_ngram_filtering=unit_generation_ngram_filtering,
                                           duration_factor=duration_factor, prosody_encoder_input=prosody_encoder_input)
        if output_modality == Modality.TEXT:
            return texts, None
        assert units is not None and self.model.t2u_model is not None
        pad_idx = self.model.t2u_model.target_vocab_info.pad_idx
        if isinstance(self.model.t2u_model, UnitYT2UModel):
            return texts, self._speech_output_ar(units, self._tls.generator.last_unit_output["unit_lens"], tgt_lang, spkr,
                                                 sample_rate)
        # translator.py:396-404 incl. the quirk that a genuine unit 1 is dropped like a pad (SURVEY a16)
        units_host = units.cpu()
        speech_units = [u[u != pad_idx].tolist() for u in units_host]
        audio_wavs: List[Tensor] = []
        if self.vocoder is not None:
            wav = self.vocoder(units, tgt_lang, spkr, dur_prediction=False)
            for i in range(len(units)):
                n = int(wav.size(-1) * len(speech_units[i]) / len(units[i]))
                audio_wavs.append(wav[i, :, :n].unsqueeze(0))
        return texts, BatchedSpeechOutput(units=speech_units, audio_wavs=audio_wavs, sample_rate=sample_rate)

    def _speech_output_ar(self, units: Tensor, unit_lens: List[int], tgt_lang: str, spkr: Optional[int],
                          sample_rate: int) -> BatchedSpeechOutput:
        """translator.py:386-428 for the AR T2U: the language token is dropped, `speech_units` loses every 1 (the pad
        quirk), and the vocoder predicts durations.  Row b is what the reference returns for that row alone at batch 1
        (it cannot vocode a batch whose rows expand to different lengths): the vocoder input is the row's own units, its
        EOS-turned-1 included, without padding, and the waveform is trimmed to
        int(hop * T_b * len(speech_units_b) / len(units_b)) of its own hop * T_b samples.  Rows with the same number of
        units are vocoded together; each row of such a batch equals the row vocoded alone."""
        pad_idx = self.model.t2u_model.target_vocab_info.pad_idx
        rows = [units[i, 1:n].cpu() for i, n in enumerate(unit_lens)]
        speech_units = [r[r != pad_idx].tolist() for r in rows]
        audio_wavs: List[Tensor] = []
        if self.vocoder is not None:
            wavs: List[Optional[Tensor]] = [None] * len(rows)
            for n in sorted({r.numel() for r in rows}):
                idx = [i for i, r in enumerate(rows) if r.numel() == n]
                wav = self.vocoder(torch.stack([rows[i] for i in idx]).to(self.device), tgt_lang, spkr, dur_prediction=True)
                for j, i in enumerate(idx):
                    keep = int(int(self.vocoder.last_wav_lens[j]) * len(speech_units[i]) / n)
                    wavs[i] = wav[j, :, :keep].unsqueeze(0)
            audio_wavs = cast(List[Tensor], wavs)
        return BatchedSpeechOutput(units=speech_units, audio_wavs=audio_wavs, sample_rate=sample_rate)
