#!/usr/bin/env python
"""Generates tests/golden/transcriber.json by EXECUTING the reference's own code here (needs the reference tree;
nothing is copied): `Transcriber._extract_timestamps`, `Transcriber.generate_lis` and
`Transcriber._collect_word_level_stats` (inference/transcriber.py:178-267).  The module is imported with type-only
stand-ins for fairseq2, the Demucs and Silero modules and the reference's model / tokenizer packages; numpy and scipy are
the real ones.

Inputs:
  * crafted attention matrices (the reference's input layout: n + 1 rows, the first dropped, and S = F + 2 columns, the
    first and last dropped): exact ties inside columns and between LIS lengths, n = 1, F = 1, a column argmax that runs
    backwards, each at filter widths 1, 3, 5 and 7;
  * random matrices up to n = 200 tokens x F = 250 frames from `oracle_transcriber.random_attention(seed, n, S)`, stored
    by seed only;
  * pair lists for generate_lis with ties;
  * piece / time / score lists for the word grouping: leading "▁", non-increasing times, empty pieces.
Start bins are read back exactly by calling _extract_timestamps with audio_len = F (one second per bin).
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

REF = "/root/reference/src/seamless_communication/inference/transcriber.py"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle_transcriber import random_attention  # noqa: E402

WIDTHS = (1, 3, 5, 7)
RANDOM = [(1, 1, 3), (2, 5, 20), (3, 17, 126), (4, 60, 126), (5, 200, 252), (6, 128, 60), (7, 3, 251), (8, 41, 9)]


class _Any:
    def __init__(self, *a, **kw):
        pass


def _stub(name):
    m = types.ModuleType(name)
    m.__getattr__ = lambda attr: type(attr, (_Any,), {})  # every imported name is a placeholder class
    m.__path__ = []
    sys.modules[name] = m
    return m


def load_reference():
    for name in ("fairseq2", "fairseq2.assets", "fairseq2.assets.card", "fairseq2.data", "fairseq2.data.audio",
                 "fairseq2.generation", "fairseq2.memory", "fairseq2.models", "fairseq2.models.nllb",
                 "fairseq2.models.nllb.tokenizer", "fairseq2.nn", "fairseq2.nn.transformer",
                 "fairseq2.nn.transformer.multihead_attention", "fairseq2.typing", "seamless_communication",
                 "seamless_communication.denoise", "seamless_communication.denoise.demucs", "seamless_communication.models",
                 "seamless_communication.models.tokenizer", "seamless_communication.models.unity",
                 "seamless_communication.segment", "seamless_communication.segment.silero_vad"):
        _stub(name)
    spec = importlib.util.spec_from_file_location("ref_transcriber", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.Transcriber


def crafted():
    """(name, rows) in the reference's layout; every column has a nonzero sum."""
    cases = []
    # ties inside columns: equal maxima in several rows
    t = np.array([[9, 9, 9, 9, 9, 9, 9],
                  [0, 2, 2, 1, 0, 0, 0],
                  [0, 2, 2, 2, 1, 1, 0],
                  [0, 1, 2, 2, 2, 1, 0],
                  [0, 0, 0, 1, 2, 2, 0]], dtype=np.float32)
    cases.append(("column_ties", t))
    # ties between LIS lengths: two increasing runs of the same length
    t = np.zeros((5, 10), dtype=np.float32)
    t[0] = 1
    for j, k in enumerate([0, 1, 0, 1, 2, 3, 2, 3]):
        t[1 + k, 1 + j] = 4
    t[1:, 1:-1] += 0.25
    cases.append(("lis_ties", t))
    # one token
    cases.append(("n1", np.array([[5, 1, 2, 3, 4], [1, 2, 3, 4, 5]], dtype=np.float32)))
    # one frame
    cases.append(("F1", np.array([[1, 1, 1], [1, 2, 1], [1, 3, 1], [1, 2, 1]], dtype=np.float32)))
    # argmax running backwards (anti-diagonal), then forwards
    t = np.full((7, 14), 0.5, dtype=np.float32)
    for j in range(12):
        t[1 + (5 - j if j < 6 else j - 6), 1 + j] = 6
    cases.append(("backwards", t))
    # dyadic values with exact ties after normalisation
    t = np.array([[0.5, 0.25, 0.25, 0.5, 0.125, 1],
                  [0.25, 0.5, 0.25, 0.125, 0.5, 0.5],
                  [0.125, 0.25, 0.5, 0.5, 0.25, 0.25],
                  [1, 0.25, 0.125, 0.25, 0.5, 0.125]], dtype=np.float32)
    cases.append(("dyadic", t))
    return cases


def main():
    T = load_reference()
    out = {"timestamps": [], "random": [], "lis": [], "words": []}

    def run(rows, w):
        F = rows.shape[1] - 2
        attn = [[float(x) for x in r] for r in rows]
        bins = T._extract_timestamps(attn, float(F), w)
        times = T._extract_timestamps(attn, 3.7, w)
        return [int(b) for b in bins], times

    for name, rows in crafted():
        for w in WIDTHS:
            bins, times = run(rows, w)
            out["timestamps"].append(dict(name=name, width=w, rows=rows.tolist(), bins=bins, times_3_7s=times))
    for seed, n, S in RANDOM:
        rows = random_attention(seed, n, S)
        for w in (3, 7) if n * S < 20000 else (3,):
            bins, times = run(rows, w)
            out["random"].append(dict(seed=seed, n=n, S=S, width=w, bins=bins, times_3_7s=times))
    for arr in ([(0, 0), (1, -1), (0, -2), (1, -3), (2, -4)], [(2, 0), (1, -1), (0, -2)], [(0, 0)],
                [(1, 0), (0, -1), (1, -2), (2, -3), (0, -4), (1, -5), (2, -6)], [(3, 0), (3, -1), (3, -2)]):
        m, seq = T.generate_lis(arr)
        out["lis"].append(dict(arr=[list(p) for p in arr], max=int(m), seq=[[int(a), int(b)] for a, b in seq]))
    for pieces, times, scores in (
            (["▁Hel", "lo", "▁world", "▁!"], [0.0, 0.2, 0.5, 0.5], [-0.1, -0.2, -0.3, -0.4]),
            (["lo", "▁a", "", "▁b", "▁c", "d"], [0.3, 0.1, 0.4, 0.4, 0.9, 0.2], [-1.0, -0.5, -0.25, 0.0, -3.0, -0.125]),
            (["▁", "▁x", "▁▁y", "z"], [0.0, 0.0, 1.0, 2.0], [-0.7, -0.01, -2.5, -0.3]),
            ([], [], [])):
        words = T._collect_word_level_stats(pieces=pieces, token_timestamps=times, step_scores=scores)
        out["words"].append(dict(pieces=pieces, times=times, scores=scores,
                                 out=[[w.text, float(w.time_s), float(w.prob)] for w in words]))
    with open(os.path.join(HERE, "transcriber.json"), "w") as f:
        json.dump(out, f, indent=None, separators=(",", ":"))


if __name__ == "__main__":
    main()
