"""Vocoder facade (reference models/vocoder/vocoder.py:15-49) over the CUDA Code-HiFiGAN engine."""
from __future__ import annotations

import threading
from typing import Any, Dict, List, Optional, Union

import torch
from torch import Tensor

from ... import config as cfgmod
from ... import synthetic as synthetic_mod
from ...engine import VocoderEngine


class Vocoder:
    def __init__(self, engine: VocoderEngine, lang_spkr_idx_map: Dict[str, Any]):
        self.code_generator = engine
        self.lang_spkr_idx_map = lang_spkr_idx_map
        self._tls = threading.local()  # LanePool workers vocode concurrently: each thread sees its own last call

    @property
    def last_wav_lens(self) -> Optional[Tensor]:
        """(N,) int64 samples per row of this thread's last dur_prediction=True call."""
        return getattr(self._tls, "wav_lens", None)

    def eval(self):
        return self

    def forward(self, units: Tensor, lang_list: Union[List[str], str], spkr_list: Union[Optional[List[int]], int] = None,
                dur_prediction: bool = True) -> Tensor:
        """Same argument conventions as the reference's Vocoder.forward (models/vocoder/vocoder.py:25-49): a single
        language / speaker applies to the whole batch, speaker -1 (or None) selects the language's first speaker.

        dur_prediction=True (the reference's default, for deduplicated units) repeats each unit by the duration the
        vocoder's own predictor gives it.  Rows may then differ in length: the output is (N, 1, hop * max_b T_b), row b
        is zero past its own hop * T_b samples, and `last_wav_lens` holds those per-row sample counts.  It needs a
        vocoder loaded with its duration predictor (code_generator.dur_predictor.*); without one it raises
        NotImplementedError."""
        if units.dim() == 1:
            units = units[None]
        n = units.size(0)
        langs = [lang_list] * n if isinstance(lang_list, str) else list(lang_list)
        if spkr_list is None or (not isinstance(spkr_list, int) and len(spkr_list) == 0):
            spkrs = [-1] * len(langs)
        else:
            spkrs = [spkr_list] * n if isinstance(spkr_list, int) else list(spkr_list)
        table = self.lang_spkr_idx_map
        lang_ids = [table["multilingual"][name] for name in langs]
        spkr_ids = [table["multispkr"][name][0] if s == -1 else s for name, s in zip(langs, spkrs)]
        if dur_prediction:
            if not getattr(self.code_generator, "has_dur_predictor", False):
                raise NotImplementedError("dur_prediction=True needs a vocoder loaded with its duration predictor "
                                          "(code_generator.dur_predictor.*)")
            wav, self._tls.wav_lens, _ = self.code_generator.resynthesize(units.reshape(n, -1), lang_ids, spkr_ids)
            return wav
        return self.code_generator(units.reshape(n, -1), lang_ids, spkr_ids)

    __call__ = forward


def load_vocoder_model(name_or_arch: str, device="cuda", dtype=torch.float16, state_dict=None, seed: int = 1, checkpoint=None,
                       synthetic: bool = False) -> Vocoder:
    """Weights: `state_dict` ("code_generator.*" keys), or `checkpoint` (path / mapping, {"generator": ...} of the original
    release or {"model": ...}; models/checkpoint.py), or `synthetic=True` for seeded random-init weights.  Without any of
    them a RuntimeError is raised instead of silently vocoding with random weights.  The language / speaker table is the
    card's: `vocoder_36langs` (seamlessM4T_large) has its own speaker ids, every other name gets vocoder_v2's."""
    arch = cfgmod.VOCODER_CARDS.get(name_or_arch, name_or_arch)
    if arch not in cfgmod.VOCODER_ARCHS:
        raise ValueError(f"unknown vocoder card / architecture '{name_or_arch}'")
    cfg = cfgmod.VOCODER_ARCHS[arch]()
    if state_dict is None and checkpoint is not None:
        from ..checkpoint import convert_vocoder_checkpoint, load_checkpoint_file
        ck = load_checkpoint_file(checkpoint) if isinstance(checkpoint, str) else checkpoint
        state_dict = convert_vocoder_checkpoint(ck)["model"]
    if state_dict is None:
        if not synthetic:
            raise RuntimeError(f"no weights for vocoder '{name_or_arch}': pass state_dict=..., checkpoint=... or synthetic=True")
        # vocoder_36langs serves seamlessM4T_large's deduplicated units: its checkpoint carries the duration predictor
        state_dict = synthetic_mod.make_vocoder_state_dict(cfg, seed=seed, dur_predictor=name_or_arch == "vocoder_36langs")
    return Vocoder(VocoderEngine(cfg, state_dict, device=device), cfgmod.vocoder_lang_spkr_idx_map(name_or_arch))
