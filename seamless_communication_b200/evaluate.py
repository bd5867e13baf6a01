"""Batched driver around `Translator.predict`: the reference's only batched caller of the hot path,
`cli/m4t/evaluate/evaluate.py` (`build_data_pipeline` :116-202, `run_eval` :248-366), SURVEY 8f row 1.

Same inputs and outputs as the reference:
    manifest      TSV with a header row (columns `audio`, the reference-text column `ctx.ref_field`, ...) or the JSON-lines
                  manifest of `m4t_prepare_dataset` (source.audio_local_path / target.text)               evaluate.py:121-143
    audio         files under `audio_root_dir`, decoded to fp32, fbank on the device                      evaluate.py:147-170
    batches       consecutive buckets of `batch_size` examples in file order, padded to the longest       evaluate.py:194-198
    corrupt input (undecodable file / NaN samples): dropped from the batch, dummy outputs written
                  (empty text, no units, one second of silence)                                           evaluate.py:204-244,281-291
    outputs       <output_path>/<stem>/model-outputs-<stem>.txt  (ref_tgt_text \\t pred_tgt_text [\\t pred_tgt_audio])
                  <output_path>/<stem>/unit_output-<stem>.txt, <output_path>/<stem>/waveform_<stem>/<id>_pred.wav
                  a RuntimeError of predict ("returned no hypothesis") skips the batch                    evaluate.py:293-311
design instead of the reference's fairseq2 DataPipeline: a small host thread pool decodes audio ahead of the GPU
(the reference maps with 4 parallel calls and prefetches 4 batches), the waveforms of a bucket go to the device as one
padded tensor + lengths, fbank runs there (`Translator.fbank_batch`), and the buckets are spread over
`parallel.LanePool` lanes so that several batches are in flight per GPU; results are written in file order.
Quality metrics (`compute_quality_metrics`: whisper ASR-BLEU, sacrebleu) need packages that are not available offline
and are out of scope; the written files are the ones that step reads.  Text-input tasks need the text encoder (out of
scope, DESIGN 7) and raise NotImplementedError."""
from __future__ import annotations

import concurrent.futures
import json
import logging
import struct
from dataclasses import dataclass, field
from pathlib import Path
from typing import Dict, Iterator, List, Optional, Tuple

import numpy as np
import torch

from .inference.generator import SequenceGeneratorOptions
from .inference.translator import BatchedSpeechOutput, Modality

logger = logging.getLogger(__name__)

SAMPLE_RATE = 16000


@dataclass
class EvalContext:
    """evaluate.py:57-108 (same field names)."""
    task: str
    data_file: Path
    audio_root_dir: Optional[Path]
    target_lang: str
    output_path: Path
    input_modality: Modality = Modality.SPEECH
    output_modality: Modality = Modality.SPEECH
    source_lang: Optional[str] = None
    batch_size: int = 4  # the reference's default (evaluate.py:413)
    ref_field: str = "tgt_text"
    text_generation_opts: SequenceGeneratorOptions = field(default_factory=SequenceGeneratorOptions)
    unit_generation_opts: Optional[SequenceGeneratorOptions] = None
    unit_generation_ngram_filtering: bool = False
    n_parallel: int = 4  # host threads decoding audio (evaluate.py:146)

    @property
    def data_file_type(self) -> str:
        return "JSON" if str(self.data_file).endswith((".json", ".jsonl")) else "TSV"


def read_manifest(ctx: EvalContext) -> List[Dict[str, str]]:
    """Rows of the manifest as dicts (TSV: header names; JSON lines: the four fields the reference extracts)."""
    rows: List[Dict[str, str]] = []
    with open(ctx.data_file, "r") as f:
        if ctx.data_file_type == "TSV":
            header = f.readline().rstrip("\n").split("\t")
            for line in f:
                line = line.rstrip("\n").rstrip()
                if line:
                    rows.append(dict(zip(header, line.split("\t"))))
        else:
            for line in f:
                if line.strip():
                    ex = json.loads(line)
                    rows.append({"src_text": ex["source"]["text"], "src_lang": ex["source"]["lang"],
                                 "audio": ex["source"]["audio_local_path"], "tgt_text": ex["target"]["text"]})
    for r in rows:
        if "audio" not in r or ctx.ref_field not in r:
            raise ValueError(f"manifest rows need the columns 'audio' and '{ctx.ref_field}', got {sorted(r)}")
    return rows


def decode_wav(path: Path, all_channels: bool = False) -> Optional[torch.Tensor]:
    """PCM WAV (8 / 16 / 32-bit integer or 32-bit float, any channel count, 16 kHz) -> (T,) fp32 in [-1, 1], channel 0, or
    with all_channels (C, T).  None for files that cannot be decoded (the reference's pipeline yields NaN features for
    those and drops them)."""
    try:
        with open(path, "rb") as f:
            raw = f.read()
        if raw[:4] != b"RIFF" or raw[8:12] != b"WAVE":
            return None
        pos, fmt_body, data = 12, None, None
        while pos + 8 <= len(raw):
            cid, size = raw[pos:pos + 4], struct.unpack("<I", raw[pos + 4:pos + 8])[0]
            body = raw[pos + 8:pos + 8 + size]
            if cid == b"fmt ":
                fmt_body = body
            elif cid == b"data":
                data = body
            pos += 8 + size + (size & 1)
        if fmt_body is None or len(fmt_body) < 16 or data is None:
            return None
        tag, channels, rate, _, _, bits = struct.unpack("<HHIIHH", fmt_body[:16])
        if tag == 0xFFFE and len(fmt_body) >= 26:  # WAVE_FORMAT_EXTENSIBLE: the sub-format GUID starts with the real tag
            tag = struct.unpack("<H", fmt_body[24:26])[0]
        if channels == 0:
            return None
        if rate != SAMPLE_RATE:
            raise ValueError(f"{path}: {rate} Hz audio; the model expects {SAMPLE_RATE} Hz (resampling is the caller's job)")
        if tag == 3 and bits == 32:
            x = np.frombuffer(data, dtype="<f4").astype(np.float32)
        elif tag == 1 and bits == 16:
            x = np.frombuffer(data, dtype="<i2").astype(np.float32) / 32768.0
        elif tag == 1 and bits == 32:
            x = np.frombuffer(data, dtype="<i4").astype(np.float32) / 2147483648.0
        elif tag == 1 and bits == 8:
            x = (np.frombuffer(data, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
        else:
            return None
        x = x[:len(x) // channels * channels].reshape(-1, channels)
        return torch.from_numpy(np.ascontiguousarray(x.T if all_channels else x[:, 0]))
    except (OSError, struct.error):
        return None


def write_wav_f32(path: Path, wav: torch.Tensor, sample_rate: int = SAMPLE_RATE) -> None:
    """(1, T) or (T,) fp32 -> 32-bit float WAV (what torchaudio.save writes for a float32 tensor, evaluate.py:336-340)."""
    x = wav.detach().to(torch.float32).cpu().reshape(-1).numpy().astype("<f4")
    body = x.tobytes()
    fmt = struct.pack("<HHIIHH", 3, 1, sample_rate, sample_rate * 4, 4, 32)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt) + 8 + len(body)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt)
        f.write(b"data" + struct.pack("<I", len(body)) + body)


def collate_bucket(waves: List[Optional[torch.Tensor]]) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor], List[bool]]:
    """One bucket -> (padded (n_valid, T_max) fp32, lengths (n_valid,) int32, validity of every example)."""
    valid = [w is not None and w.numel() >= 400 and bool(torch.isfinite(w).all()) for w in waves]  # < 25 ms: no fbank frame
    good = [w for w, ok in zip(waves, valid) if ok]
    if not good:
        return None, None, valid
    T = max(w.numel() for w in good)
    batch = torch.zeros((len(good), T), dtype=torch.float32)
    for i, w in enumerate(good):
        batch[i, :w.numel()] = w
    return batch, torch.tensor([w.numel() for w in good], dtype=torch.int32), valid


def adjust_output_for_corrupted_inputs(valid: List[bool], text_output: List[str], speech_output: Optional[BatchedSpeechOutput],
                                       with_speech: bool) -> Tuple[List[str], Optional[BatchedSpeechOutput]]:
    """evaluate.py:204-244: dummy outputs at the positions of the dropped examples."""
    texts: List[str] = []
    speech = BatchedSpeechOutput(units=[], audio_wavs=[]) if with_speech else None
    k = 0
    for ok in valid:
        if ok:
            texts.append(text_output[k])
            if speech is not None:
                speech.units.append(speech_output.units[k])
                speech.audio_wavs.append(speech_output.audio_wavs[k])
            k += 1
        else:
            texts.append("")
            if speech is not None:
                speech.units.append([])
                speech.audio_wavs.append(torch.zeros(1, 1, speech.sample_rate))
    return texts, speech


def iter_buckets(ctx: EvalContext, rows: List[Dict[str, str]], prefetch: int = 4) -> Iterator[Tuple[int, List[Dict[str, str]], list]]:
    """Buckets of decoded waveforms in file order; decoding runs `prefetch` buckets ahead on ctx.n_parallel threads."""
    root = Path(ctx.audio_root_dir) if ctx.audio_root_dir is not None else Path(".")
    buckets = [rows[i:i + ctx.batch_size] for i in range(0, len(rows), ctx.batch_size)]
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, ctx.n_parallel)) as ex:
        pending: List[list] = []
        nxt = 0
        for bi in range(len(buckets)):
            while nxt < len(buckets) and nxt <= bi + prefetch:
                pending.append([ex.submit(decode_wav, root / r["audio"]) for r in buckets[nxt]])
                nxt += 1
            yield bi, buckets[bi], [f.result() for f in pending.pop(0)]


def run_eval(translator, ctx: EvalContext, lanes: int = 1, n_samples: Optional[int] = None) -> Dict[str, object]:
    """Run the manifest through `translator.predict` and write the reference's output files.  Returns the paths and counts."""
    if ctx.input_modality != Modality.SPEECH:
        raise NotImplementedError("text-input evaluation needs the text encoder (outside the S2ST hot path)")
    from .parallel import LanePool

    rows = read_manifest(ctx)
    if n_samples:
        rows = rows[:n_samples]
    stem = Path(ctx.data_file).stem
    out_dir = Path(ctx.output_path) / stem
    out_dir.mkdir(parents=True, exist_ok=True)
    with_speech = ctx.output_modality == Modality.SPEECH
    wav_dir = out_dir / f"waveform_{stem}"
    if with_speech:
        wav_dir.mkdir(parents=True, exist_ok=True)
    hyp_path, unit_path = out_dir / f"model-outputs-{stem}.txt", out_dir / f"unit_output-{stem}.txt"
    device = translator.device
    engines = [translator.model.engine] if hasattr(getattr(translator, "model", None), "engine") else []
    pool = LanePool(device, max(1, lanes), engines)

    def step(batch: Optional[torch.Tensor], lens: Optional[torch.Tensor]):
        if batch is None:
            return [], (BatchedSpeechOutput(units=[], audio_wavs=[]) if with_speech else None)
        src = translator.fbank_batch(batch, lens)
        texts, speech = translator.predict(src, ctx.task, ctx.target_lang, src_lang=ctx.source_lang,
                                           text_generation_opts=ctx.text_generation_opts,
                                           unit_generation_opts=ctx.unit_generation_opts,
                                           unit_generation_ngram_filtering=ctx.unit_generation_ngram_filtering)
        if speech is not None:  # bring the waveforms to the host on the lane's stream; the writer thread only touches host memory
            speech = BatchedSpeechOutput(units=speech.units, audio_wavs=[w.float().cpu() for w in speech.audio_wavs],
                                         sample_rate=speech.sample_rate)
        return [str(t) for t in texts], speech

    sample_id = skipped = corrupted = 0
    inflight: List[tuple] = []

    def drain_one(hyp_file, unit_file):
        nonlocal sample_id, skipped
        fut, bucket, valid = inflight.pop(0)
        try:
            (texts, speech), _ = fut.result()
        except RuntimeError as e:  # "The sequence generator returned no hypothesis ...": the reference logs and moves on
            logger.exception(f"Caught RuntimeError: {e}")
            skipped += len(bucket)
            return
        if not all(valid):
            texts, speech = adjust_output_for_corrupted_inputs(valid, texts, speech, with_speech)
        for i, row in enumerate(bucket):
            if with_speech:
                unit_file.write(" ".join(str(u) for u in speech.units[i]) + "\n")
                wav_fp = wav_dir / f"{sample_id}_pred.wav"
                write_wav_f32(wav_fp, speech.audio_wavs[i], speech.sample_rate)
                hyp_file.write(f"{row[ctx.ref_field]}\t{texts[i]}\t{wav_fp}\n")
            else:
                hyp_file.write(f"{row[ctx.ref_field]}\t{texts[i]}\n")
            sample_id += 1

    try:
        with open(hyp_path, "w") as hyp_file, open(unit_path if with_speech else "/dev/null", "w") as unit_file:
            hyp_file.write("ref_tgt_text\tpred_tgt_text\tpred_tgt_audio\n" if with_speech else "ref_tgt_text\tpred_tgt_text\n")
            for bi, bucket, waves in iter_buckets(ctx, rows):
                batch, lens, valid = collate_bucket(waves)
                if not all(valid):
                    corrupted += valid.count(False)
                    logger.warning(f"Sample IDs {bi * ctx.batch_size} to {bi * ctx.batch_size + len(bucket)} has some corrupted input.")
                inflight.append((pool.submit(bi, step, batch, lens), bucket, valid))
                if len(inflight) >= pool.lanes:
                    drain_one(hyp_file, unit_file)
            while inflight:
                drain_one(hyp_file, unit_file)
    finally:
        pool.close()
    logger.info(f"Processed {sample_id} samples")
    return {"model_outputs": hyp_path, "unit_outputs": unit_path if with_speech else None,
            "waveforms_dir": wav_dir if with_speech else None, "samples": sample_id, "skipped": skipped, "corrupted": corrupted}
