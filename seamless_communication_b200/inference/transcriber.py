"""`Transcriber`: speech recognition with word timestamps (behavioural mirror of reference inference/transcriber.py:63-428).

The reference hooks the last decoder layer's encoder-decoder attention, keeps its weights at every search step, moves
them to the host and derives each token's start time there (medfilt2d + a pure-Python longest increasing subsequence),
one utterance at a time.  Here the search records the head-summed weights on the device (sb_decode_cross_attn_weights),
the winner's rows are gathered along its cache slots and the start bins come from one kernel for the whole batch
(sb_token_timestamps); only the word grouping runs on the host.  DESIGN.md section 13 lists the deviations."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from ..models.unity import UnitYModel, load_unity_model
from .translator import Modality, Translator

SAMPLE_RATE = 16000
MAX_FILTER_WIDTH = 7  # SB_TS_MAX_WIDTH of sb_token_timestamps
# fairseq2 0.2 BeamSearchSeq2SeqGenerator defaults of the options the reference passes through [fs2-recall]
GENERATOR_DEFAULTS = dict(beam_size=1, min_gen_len=1, max_gen_len=(1, 128), max_seq_len=1024, len_penalty=1.0, unk_penalty=0.0)


@dataclass
class TranscriptionTokenStats:
    """A word while it is being assembled: its text so far, its start time and the exp(score) of each piece."""
    text: str
    time_s: float
    scores: List[float]


@dataclass
class TranscriptionToken:
    """One word of a transcription: its text, its start time in seconds and the mean probability of its pieces."""
    text: str
    time_s: float
    prob: float


class Transcription:
    """The words of one utterance (`tokens`) and their text joined by single spaces (`text`, also str() and repr())."""

    def __init__(self, tokens: List[TranscriptionToken]):
        self.tokens = tokens
        self.text = " ".join(word.text for word in tokens)

    def __add__(self, other: "Transcription") -> "Transcription":
        """Appends `other` to this transcription in place and returns it (the reference's semantics)."""
        self.tokens.extend(other.tokens)
        self.text = f"{self.text} {other.text}"
        return self

    def __str__(self) -> str:
        return self.text

    __repr__ = __str__


def _generator_options(opts: Dict) -> Dict:
    unknown = sorted(set(opts) - set(GENERATOR_DEFAULTS))
    if unknown:
        raise TypeError(f"unexpected sequence generator option(s): {', '.join(unknown)}")
    o = {**GENERATOR_DEFAULTS, **{k: v for k, v in opts.items() if v is not None}}
    o["beam_size"] = o["beam_size"] or 1  # transcriber.py:280
    return o


def _check_filter_width(filter_width: int) -> None:
    if filter_width < 1 or filter_width % 2 == 0:
        raise ValueError("Each element of kernel_size should be odd.")  # scipy.signal.medfilt2d's error
    if filter_width > MAX_FILTER_WIDTH:
        raise ValueError(f"filter_width {filter_width} is above {MAX_FILTER_WIDTH}, the widest median filter of sb_token_timestamps")


class Transcriber:
    def __init__(self, model_name_or_card: Union[str, UnitYModel], device: Union[str, torch.device] = "cuda",
                 dtype: torch.dtype = torch.float32, *, state_dict=None, checkpoint=None, synthetic: bool = False,
                 tokenizer=None):
        """Loads the model as `Translator` does (speech encoder and text decoder only).  `tokenizer`: the
        (text tokenizer, char tokenizer) pair the weights belong to; the NLLB text tokenizer is used whatever the card
        (the reference reads a `tokenizer_type` field that no seamlessM4T card has).  The kernels store fp16 and
        accumulate in fp32 whatever `dtype` says."""
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("seamless_communication_b200.Transcriber needs a CUDA device (sm_90a); no CPU fallback exists.")
        self.dtype = dtype
        if isinstance(model_name_or_card, UnitYModel):
            self.model = model_name_or_card
        else:
            self.model = load_unity_model(model_name_or_card, device=self.device, dtype=torch.float16, state_dict=state_dict,
                                          checkpoint=checkpoint, synthetic=synthetic, tokenizers=tokenizer, with_t2u=False)
        self.model.eval()
        self.engine = self.model.engine
        self.tokenizer = self.engine.text_tokenizer
        self._frontend = Translator(self.model, None, self.device, output_modality=Modality.TEXT)  # its device fbank batch

    # -- the reference's static steps ----------------------------------------------------------------------------------
    @classmethod
    def _collect_word_level_stats(cls, pieces: List[str], token_timestamps: List[float],
                                  step_scores: List[float]) -> List[TranscriptionToken]:
        """A piece opens a new word when it is the first, or starts with "▁" at a later time than the current word;
        otherwise it is appended.  A word's probability is the mean of exp(score) over its pieces."""
        assert len(pieces) == len(token_timestamps) == len(step_scores)
        stats: List[TranscriptionTokenStats] = []
        for piece, time_s, score in zip(pieces, token_timestamps, step_scores):
            prob = np.exp(score)
            if stats and not (piece.startswith("▁") and time_s > stats[-1].time_s):
                stats[-1].text += piece.replace("▁", " ")
                stats[-1].scores.append(prob)
            else:
                stats.append(TranscriptionTokenStats(piece.replace("▁", " ").strip(), time_s, [prob]))
        return [TranscriptionToken(s.text, s.time_s, np.mean(s.scores).item()) for s in stats]

    # -- input ---------------------------------------------------------------------------------------------------------
    @staticmethod
    def _waveform(audio: Union[str, Tensor], sample_rate: int) -> Tensor:
        """(T,) fp32 of a WAV path or a (T,) / (T, 1) tensor."""
        if sample_rate != SAMPLE_RATE:
            raise ValueError(f"sample_rate {sample_rate} is not supported: the fbank frontend takes {SAMPLE_RATE} Hz (no resampling)")
        if isinstance(audio, str):
            from ..evaluate import decode_wav
            wav = decode_wav(audio, all_channels=True)
            if wav is None:
                raise ValueError(f"{audio}: not a {SAMPLE_RATE} Hz PCM WAV file")
            wav = wav.t()
        else:
            wav = audio
        if wav.dim() == 2 and wav.size(1) == 1:
            wav = wav[:, 0]
        if wav.dim() != 1:
            raise ValueError(f"audio of shape {tuple(wav.shape)}: one channel is supported, as (T,) or (T, 1)")
        return wav.to(torch.float32)

    # -- transcription -------------------------------------------------------------------------------------------------
    @torch.inference_mode()
    def transcribe(self, audio: Union[str, Tensor], src_lang: str, filter_width: int = 3, sample_rate: int = SAMPLE_RATE,
                   denoise: bool = False, denoise_config=None, chunk_size_sec: int = 20, pause_length_sec: float = 1,
                   **sequence_generator_options) -> Transcription:
        """Transcribes one utterance: every word with its start time and mean token probability.  Inputs longer than
        `chunk_size_sec` raise ValueError (the reference splits them with the Silero VAD, which is not available), and
        `denoise=True` raises NotImplementedError (Demucs is not available)."""
        if denoise:
            raise NotImplementedError("denoise=True needs Demucs, which is not available")
        _check_filter_width(filter_width)
        opts = _generator_options(sequence_generator_options)
        wav = self._waveform(audio, sample_rate)
        if wav.numel() / sample_rate > chunk_size_sec:
            raise ValueError(f"audio of {wav.numel() / sample_rate:.2f} s is longer than chunk_size_sec={chunk_size_sec}: "
                             "segmenting long inputs needs the Silero VAD, which is not available")
        # the reference encodes the fbank of this waveform alone, without a padding mask (its frontend drops an odd frame)
        fb = self._frontend.fbank_batch(wav[None])
        frames = int(fb["seq_lens"][0])
        return self._run(fb["seqs"][:, :frames - frames % 2], None, [wav.numel() / sample_rate], src_lang, filter_width, opts)[0]

    @torch.inference_mode()
    def transcribe_batch(self, audios: List[Union[str, Tensor]], src_lang: str, filter_width: int = 3,
                         sample_rate: int = SAMPLE_RATE, **sequence_generator_options) -> List[Transcription]:
        """`transcribe` for a list of utterances of any lengths up to 20 s: one fbank batch, one encoder pass, one search and
        one timestamp kernel.  Row b is row b transcribed alone, except that the search's length budget follows the longest
        row (as in `Translator.predict`)."""
        _check_filter_width(filter_width)
        opts = _generator_options(sequence_generator_options)
        waves = [self._waveform(a, sample_rate) for a in audios]
        if not waves:
            return []
        for w in waves:
            if w.numel() / sample_rate > 20:
                raise ValueError(f"audio of {w.numel() / sample_rate:.2f} s is longer than 20 s: segmenting long inputs needs "
                                 "the Silero VAD, which is not available")
        T = max(w.numel() for w in waves)
        batch = torch.zeros((len(waves), T), dtype=torch.float32)
        for i, w in enumerate(waves):
            batch[i, :w.numel()] = w.cpu()
        ns = torch.tensor([w.numel() for w in waves], dtype=torch.int32)
        fb = self._frontend.fbank_batch(batch, ns)
        return self._run(fb["seqs"], fb["seq_lens"], [w.numel() / sample_rate for w in waves], src_lang, filter_width, opts)

    def _run(self, fbank: Tensor, frames: Optional[Tensor], seconds: List[float], src_lang: str, filter_width: int,
             opts: Dict) -> List[Transcription]:
        eng = self.engine
        enc, enc_lens = eng.encode_speech(fbank.to(torch.float16).contiguous(), frames)
        prefix = self.tokenizer.create_encoder(task="translation", lang=src_lang, mode="target").prefix_indices.tolist()
        hyps = eng.beam_search(enc, enc_lens, prefix, beam=opts["beam_size"], soft_max=tuple(opts["max_gen_len"]),
                               hard_max=opts["max_seq_len"], len_penalty=opts["len_penalty"], unk_penalty=opts["unk_penalty"],
                               min_seq_len=opts["min_gen_len"], record_attention=True)
        stamps = eng.token_timestamps(filter_width)
        lens = enc_lens.tolist() if enc_lens is not None else [enc.T] * enc.B
        out = []
        for b, (h, (starts, scores)) in enumerate(zip(hyps, stamps)):
            if not h:  # no finished hypothesis (the reference raises IndexError here)
                out.append(Transcription([]))
                continue
            ids = h[0][1][len(prefix):-1]
            F = int(lens[b]) - 2
            per_bin = seconds[b] / F if F >= 1 else 0.0
            pieces = [self.tokenizer.model.index_to_token(i) for i in ids]
            out.append(Transcription(self._collect_word_level_stats(pieces, [per_bin * s for s in starts], scores)))
        return out
