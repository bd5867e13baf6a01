"""Audio to units (reference models/unit_extractor/unit_extractor.py:37-116): an XLS-R wav2vec2 encoder up to one layer,
then the nearest of the k-means centroids per frame, on the CUDA kernels of `Wav2Vec2Engine`.

Deviation from the reference: the computation is fp16 storage with fp32 accumulation whatever `dtype` says (as for
`Translator`); the reference's `m4t_audio_to_units` CLI runs fp32.  Units of frames whose nearest two centroids lie
closer than the fp16 feature error can differ (DESIGN.md section 11).
"""
from __future__ import annotations

import os
import struct
from typing import Any, List, Mapping, Optional, Union

import numpy as np
import torch
from torch import Tensor

from ... import config as cfgmod
from ... import synthetic as synthetic_mod
from ...wav2vec2_engine import Wav2Vec2Engine

KMEANS_10K_SHAPE = (10000, 1280)  # kmeans_10k.npy holds (K, dim); KmeansModel transposes it on load (kmeans.py:17-19)
SAMPLE_RATE = 16000


def _wav_channels(path: str) -> int:
    """Channel count from a RIFF/WAVE header (0 when there is no fmt chunk)."""
    with open(path, "rb") as f:
        raw = f.read(4096)
    pos = 12
    while pos + 8 <= len(raw):
        cid, size = raw[pos:pos + 4], struct.unpack("<I", raw[pos + 4:pos + 8])[0]
        if cid == b"fmt " and pos + 12 <= len(raw):
            return struct.unpack("<H", raw[pos + 10:pos + 12])[0]
        pos += 8 + size + (size & 1)
    return 0


class UnitExtractor:
    """Unit extractor which converts raw audio into units.

    model_name_or_card: "xlsr2_1b_v2" (or a test copy of it, config.WAV2VEC2_ARCHS).  Weights: `state_dict` (fairseq2
    names), `checkpoint` (path or mapping of the fairseq `xlsr2_1b_v2.pt`, models/checkpoint.py) or `synthetic=True`
    for seeded random-init weights; without any of them a RuntimeError is raised.  kmeans_uri: a local `.npy` of shape
    (K, model_dim), as the reference's kmeans_10k.npy; nothing is downloaded, so a URL raises ValueError.  With
    synthetic=True and no file, `kmeans_uri` may be None and K = num_centroids seeded centroids are drawn."""

    def __init__(self, model_name_or_card: str, kmeans_uri: Optional[str], device: Union[str, torch.device] = "cuda",
                 dtype: torch.dtype = torch.float32, *, state_dict: Optional[Mapping[str, Tensor]] = None,
                 checkpoint: Union[str, Mapping[str, Any], None] = None, synthetic: bool = False, seed: int = 3,
                 num_centroids: int = 10000):
        if model_name_or_card not in cfgmod.WAV2VEC2_ARCHS:
            raise ValueError(f"unknown wav2vec2 model '{model_name_or_card}' (known: {sorted(cfgmod.WAV2VEC2_ARCHS)})")
        cfg = cfgmod.WAV2VEC2_ARCHS[model_name_or_card]()
        if kmeans_uri is not None and "://" in kmeans_uri:
            raise ValueError(f"kmeans_uri '{kmeans_uri}' is a URL; nothing is downloaded: pass a local .npy file")
        if kmeans_uri is not None:
            centroids = torch.from_numpy(np.ascontiguousarray(np.load(kmeans_uri))).float()
        elif synthetic:
            centroids = synthetic_mod.make_kmeans_centroids(num_centroids, cfg.model_dim, seed=seed + 1)
        else:
            raise ValueError("kmeans_uri is required unless synthetic=True")
        if centroids.dim() != 2 or centroids.shape[1] != cfg.model_dim:
            raise ValueError(f"k-means centroids have width {tuple(centroids.shape)[1:]}, the model's features {cfg.model_dim}")
        if state_dict is None and checkpoint is not None:
            from ..checkpoint import convert_wav2vec2_checkpoint, load_checkpoint_file
            ck = load_checkpoint_file(checkpoint) if isinstance(checkpoint, str) else checkpoint
            state_dict = convert_wav2vec2_checkpoint(ck)["model"]
        if state_dict is None:
            if not synthetic:
                raise RuntimeError(f"no weights for '{model_name_or_card}': pass state_dict=..., checkpoint=... or synthetic=True")
            state_dict = synthetic_mod.make_wav2vec2_state_dict(cfg, seed=seed)
        self.cfg = cfg
        self.device = torch.device(device)
        self.dtype = dtype
        self.engine = Wav2Vec2Engine(cfg, dict(state_dict), centroids, device=self.device)

    def _check_layer(self, out_layer_idx: int) -> None:
        if not 0 <= out_layer_idx < self.cfg.num_encoder_layers:
            raise ValueError(f"out_layer_idx {out_layer_idx} is outside [0, {self.cfg.num_encoder_layers})")

    @torch.inference_mode()
    def predict(self, audio: Union[str, Tensor], out_layer_idx: int, sample_rate: int = SAMPLE_RATE) -> Tensor:
        """Units (T,) int64 of one utterance: a WAV path (mono, 16 kHz), a 1-D tensor, or a 2-D tensor that is transposed
        when size(0) < size(1) (unit_extractor.py:78-93) and must then hold one channel; multi-channel input raises."""
        if sample_rate != SAMPLE_RATE:
            raise ValueError(f"Input audio must have {SAMPLE_RATE} sampling rate, got {sample_rate}")
        self._check_layer(out_layer_idx)
        if isinstance(audio, str):
            from ...evaluate import decode_wav
            if _wav_channels(audio) > 1:
                raise ValueError(f"{audio}: multi-channel audio; the reference would interleave the channels into one "
                                 "sequence, pass one channel")
            wav = decode_wav(audio)
            if wav is None:
                raise ValueError(f"{audio}: not a decodable PCM WAV file")
        else:
            if audio.dim() > 2:
                raise ValueError("The audio tensor can't be more than 2 dimensions.")
            wav = audio
            if wav.dim() == 2 and wav.size(0) < wav.size(1):
                wav = wav.transpose(0, 1)
            if wav.dim() == 2 and wav.size(1) != 1:
                # the reference pads T (not T * C) to even with rows of 1.0, flattens the channels into one sequence and
                # keeps a padding mask of T frames: not an interpretation of multi-channel audio worth reproducing
                raise ValueError(f"audio tensor of shape {tuple(audio.shape)} has {wav.size(1)} channels; pass one channel")
            wav = wav.reshape(-1)
        wav = wav.to(self.device, torch.float32).reshape(1, -1)
        return self.predict_batch(wav, torch.tensor([wav.shape[1]]), out_layer_idx)[0]

    @torch.inference_mode()
    def predict_batch(self, waves: Tensor, num_samples: Union[Tensor, List[int]], out_layer_idx: int = 34) -> List[Tensor]:
        """waves (N, T) fp32, row b valid up to num_samples[b] -> N unit tensors; row b equals
        predict(waves[b, :num_samples[b]]) bit for bit."""
        self._check_layer(out_layer_idx)
        if waves.dim() != 2:
            raise ValueError("waves must be (N, T)")
        ns = [int(n) for n in (num_samples.tolist() if isinstance(num_samples, Tensor) else num_samples)]
        if len(ns) != waves.shape[0]:
            raise ValueError(f"{len(ns)} sample counts for {waves.shape[0]} rows")
        feats, n_out = self.engine.forward(waves, ns, out_layer_idx)
        return self.engine.units(feats, n_out)

    @staticmethod
    def resynthesize_audio(units: Tensor, src_lang: str, device, dtype=torch.float16, vocoder_name: str = "vocoder_v2",
                           **vocoder_kwargs) -> Tensor:
        """vocoder(units, src_lang, spkr=-1, dur_prediction=True) on the project's Vocoder (unit_extractor.py:100-116);
        `vocoder_kwargs` (state_dict= / checkpoint= / synthetic=) reach load_vocoder_model."""
        from ..vocoder import load_vocoder_model
        vocoder = load_vocoder_model(vocoder_name, device=device, dtype=dtype, **vocoder_kwargs)
        return vocoder(units, src_lang, -1, dur_prediction=True)
