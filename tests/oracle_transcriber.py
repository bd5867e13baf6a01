"""CPU oracle of the transcriber (reference inference/transcriber.py), test infrastructure like oracle/unity_oracle.py.

`UnityOracleTranscriber` subclasses `UnityOracle` and leaves its pinned search untouched: its `beam_search` is the same
search step for step, and it also records, for every hypothesis, the last decoder layer's head-summed cross-attention
weights at each position and its cumulative scores (what the reference's AttentionWeightHook and fairseq2's step scores
give).  The timestamp algorithm and the word grouping are restated here in float64 numpy (tests/golden/transcriber.json
holds what the reference's own functions return on the same inputs):

  1. A[k][j] = W[P-1+k][1+j], k < n generated tokens, j < F = S - 2 frames (the reference's [:-1], [1:] and [1:-1]);
  2. columns divided by their sum over k = 0 .. n-1 in that order; a zero column becomes 0 (the reference: NaN);
  3. a w x w median filter, zero padding (scipy.signal.medfilt2d; w must be odd);
  4. per column the smallest k attaining the maximum (np.argmax);
  5. generate_lis over (c[j], -j): L[i] = 1 + max L[j] over j < i with c[j] < c[i], prev[i] the first such j attaining it
     (i when none), the path ending at the first i of largest L;
  6. start[c] = j along the path, other tokens the previous start (token 0: 0);
  7. time = start * (seconds / F).
Per-token scores are float32(cum[P+k] - cum[P+k-1]) [fs2-recall: fairseq2 0.2 turns the cumulative scores into step
scores by differencing], probabilities exp(score) in float64.
"""
from __future__ import annotations

import math
import os
import sys
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.unity_oracle import UnityOracle, key_mask  # noqa: E402


# ------------------------------------------------------------------------------------------------ inputs of the fixture
def random_attention(seed: int, n: int, S: int) -> np.ndarray:
    """(n + 1, S) float32 rows shaped like head-summed attention (peaked, positive): the reference's input layout
    (its first row and first / last columns are dropped)."""
    rng = np.random.default_rng(seed)
    return (rng.random((n + 1, S)) ** 6 * 4.0).astype(np.float32)


# ------------------------------------------------------------------------------------------------ restatement
def lis(c: List[int]) -> Tuple[List[int], List[int], int]:
    """Steps 5 on the column argmaxes c: (L, prev, end)."""
    F = len(c)
    ca = np.asarray(c, dtype=np.int64)
    L = np.ones(F, dtype=np.int64)
    prev = list(range(F))
    for i in range(1, F):
        cand = np.where(ca[:i] < ca[i], L[:i], 0)
        best = int(cand.max())
        if best > 0:
            L[i], prev[i] = best + 1, int(np.argmax(cand))  # argmax: the first j attaining it
    return L.tolist(), prev, int(np.argmax(L))


def start_bins(A: np.ndarray, width: int) -> List[int]:
    """Steps 2-6 on A (n, F) float64."""
    if width < 1 or width % 2 == 0:
        raise ValueError("Each element of kernel_size should be odd.")
    n, F = A.shape
    s = np.zeros(F)
    for k in range(n):
        s = s + A[k]
    A = np.where(s != 0, A / np.where(s != 0, s, 1.0), 0.0)
    r = width // 2
    pad = np.zeros((n + 2 * r, F + 2 * r))
    pad[r:r + n, r:r + F] = A
    win = np.lib.stride_tricks.sliding_window_view(pad, (width, width)).reshape(n, F, width * width)
    filt = np.sort(win, axis=-1)[:, :, (width * width) // 2]
    c = [int(x) for x in filt.argmax(axis=0)]
    L, prev, i = lis(c)
    starts = [-1] * n
    starts[c[i]] = i
    while prev[i] != i:
        i = prev[i]
        starts[c[i]] = i
    last, out = 0, []
    for k in range(n):
        last = starts[k] if starts[k] >= 0 else last
        out.append(last)
    return out


def start_bins_from_rows(rows: np.ndarray, width: int) -> List[int]:
    """The reference's input layout: rows (n + 1, S) -> A = rows[1:, 1:-1] in float64."""
    return start_bins(np.asarray(rows, dtype=np.float64)[1:, 1:-1], width)


def word_stats(pieces: List[str], times: List[float], scores: List[float]) -> List[Tuple[str, float, float]]:
    """_collect_word_level_stats: (text, time_s, prob) per word."""
    words: List[list] = []
    for p, t, sc in zip(pieces, times, scores):
        if not words or (p.startswith("▁") and t > words[-1][1]):
            words.append([p.replace("▁", " ").strip(), t, [np.exp(sc)]])
        else:
            words[-1][0] += p.replace("▁", " ")
            words[-1][2].append(np.exp(sc))
    return [(w[0], w[1], float(np.mean(w[2]))) for w in words]


# ------------------------------------------------------------------------------------------------ search with recording
class UnityOracleTranscriber(UnityOracle):
    """`beam_search` records, per finished hypothesis (best first, in `self.records[sentence]`): `attn` (step + 1, S)
    float64, row t the head-summed softmax weights of the last layer's cross-attention at decoder position t; `cum`
    (len,) float32 cumulative scores, the EOS's unnormalised score last."""

    def __init__(self, *a, record_layer: Optional[int] = None, **kw):
        """`record_layer`: the decoder layer whose cross-attention is recorded (default the last, as the reference's hook;
        another layer serves tests as a negative control)."""
        super().__init__(*a, **kw)
        self._rec: Optional[list] = None
        layer = self.c["dec_layers"] - 1 if record_layer is None else record_layer
        self._last_cross = f"text_decoder.layers.{layer}.encoder_decoder_attn"

    def mha(self, p, q_in, kv_in, kmask=None, causal=False, rel_k=None, cache=None):
        out = super().mha(p, q_in, kv_in, kmask, causal, rel_k, cache)
        if self._rec is not None and p == self._last_cross:
            N, Sq, _ = q_in.shape
            H, K = self.H, self.M // self.H
            q = self.lin(q_in, p + ".q_proj").view(N, Sq, H, K).transpose(1, 2).double()
            if cache is not None and "k" in cache:
                k = cache["k"].double()
            else:
                k = self.lin(kv_in, p + ".k_proj").view(N, kv_in.shape[1], H, K).transpose(1, 2).double()
            w = torch.matmul(q, k.transpose(2, 3)) * (K ** -0.5)
            if kmask is not None:
                w = w.masked_fill(~kmask[:, None, None, :], float("-inf"))
            self._rec.append(torch.softmax(w, dim=-1).sum(1))  # (N, Sq, S)
        return out

    def beam_search(self, enc, enc_lens, prefix: List[int], beam=5, soft_max=(1, 200), hard_max=1024,
                    len_penalty=1.0, unk_penalty=0.0, min_seq_len=1, trace=None):
        V = self.c["text_vocab"]
        eos, pad, unk = self.c["text_eos"], self.c["text_pad"], self.c["text_unk"]
        results, self.records = [], []
        for n in range(enc.shape[0]):
            S_enc = int(enc_lens[n]) if enc_lens is not None else enc.shape[1]
            a, b = soft_max
            max_len = hard_max if a <= 0 else min(hard_max, int(a * enc.shape[1]) + b)
            e = enc[n:n + 1].expand(beam, -1, -1)
            ekm = key_mask(torch.full((beam,), S_enc), enc.shape[1]) if enc_lens is not None else None
            caches = [({}, {"static": True}) for _ in range(self.c["dec_layers"])]
            seqs = torch.zeros(beam, max_len, dtype=torch.long)
            scores = torch.zeros(beam, max_len)
            att = torch.zeros(beam, max_len, enc.shape[1], dtype=torch.float64)
            P = len(prefix)
            seqs[:, :P] = torch.tensor(prefix)
            self._rec = []
            if P > 1:
                h = self.decoder(self.embed_text(seqs[:, :P - 1], 0), e, ekm, caches)
                att[:, :P - 1] = self._rec.pop()
                lp = torch.log_softmax(self.project(h).float(), dim=-1)
                acc = 0.0
                for i in range(1, P):
                    acc = acc + float(lp[0, i - 1, prefix[i]])
                    scores[:, i] = acc
            finished: List[Dict] = []
            done = False
            for step in range(P - 1, max_len - 1):
                h = self.decoder(self.embed_text(seqs[:, step:step + 1], step), e, ekm, caches)
                att[:, step] = self._rec.pop()[:, 0]
                logits = self.project(h[:, 0])
                lp = torch.log_softmax(logits.float(), dim=-1)
                if trace is not None and n == trace.get("sentence", 0):
                    trace.setdefault("logits", []).append(logits.clone())
                    trace.setdefault("inputs", []).append(seqs[:, step].clone())
                if step < min_seq_len:
                    lp[:, eos] = -math.inf
                if step == max_len - 2:
                    lp[:, :eos] = -math.inf
                    lp[:, eos + 1:] = -math.inf
                lp[:, pad] = -math.inf
                if unk_penalty != 0:
                    lp[:, unk] -= unk_penalty
                cand = lp[0:1] + scores[0:1, step:step + 1] if step == P - 1 else lp + scores[:, step:step + 1]
                top_s, top_i = torch.topk(cand.reshape(-1), min(2 * beam, V - 1))
                bi, ti, si = [], [], []
                for c_s, c_i in zip(top_s.tolist(), top_i.tolist()):
                    bm, tok = c_i // V, c_i % V
                    if tok == eos and c_s != -math.inf:
                        cum = torch.cat([scores[bm, :step + 1], torch.tensor([c_s], dtype=torch.float32)])
                        finished.append(dict(score=c_s / float((step + 1) ** len_penalty), ids=seqs[bm, :step + 1].tolist() + [tok],
                                             attn=att[bm, :step + 1].clone(), cum=cum))
                        if len(finished) == beam:
                            done = True
                            break
                        continue
                    bi.append(bm); ti.append(tok); si.append(c_s)
                    if len(bi) >= beam:
                        break
                if done:
                    break
                bidx = torch.tensor(bi)
                seqs, scores, att = seqs[bidx].clone(), scores[bidx].clone(), att[bidx].clone()
                seqs[:, step + 1] = torch.tensor(ti)
                scores[:, step + 1] = torch.tensor(si)
                for sc, _ in caches:
                    sc["k"], sc["v"] = sc["k"][bidx], sc["v"][bidx]
                if trace is not None and n == trace.get("sentence", 0):
                    trace.setdefault("beam_idx", []).append(bidx.clone())
            self._rec = None
            order = sorted(range(len(finished)), key=lambda j: -finished[j]["score"])
            if trace is not None and n == trace.get("sentence", 0):
                trace["finished"] = [(f["score"], f["ids"]) for f in finished]
                trace["max_len"] = max_len
                trace["prefix_scores"] = scores[0, :P].clone()
            self.records.append([finished[j] for j in order])
            results.append([(finished[j]["score"], finished[j]["ids"]) for j in order])
        return results

    def transcribe(self, fb, fb_lens, seconds: List[float], prefix: List[int], width=3, beam=1, soft_max=(1, 128),
                   hard_max=1024) -> List[Dict]:
        """Per row: ids (generated, EOS excluded), filtered-matrix inputs A (n, F), start bins, scores, times, words."""
        enc, lens = self.encode_speech(fb, fb_lens)
        self.beam_search(enc, lens, prefix, beam=beam, soft_max=soft_max, hard_max=hard_max)
        P, out = len(prefix), []
        for b, recs in enumerate(self.records):
            if not recs:
                out.append(dict(ids=[], bins=[], scores=[], times=[], A=None, F=0))
                continue
            r = recs[0]
            ids = r["ids"][P:-1]
            n = len(ids)
            S = int(lens[b]) if lens is not None else enc.shape[1]
            F = S - 2
            A = r["attn"][P - 1:P - 1 + n, 1:1 + F].numpy()
            bins = start_bins(A, width) if n > 0 and F >= 1 else [0] * n
            cum = r["cum"]
            scores = (cum[P:P + n] - cum[P - 1:P - 1 + n]).tolist()
            per_bin = seconds[b] / F if F >= 1 else 0.0
            out.append(dict(ids=ids, bins=bins, scores=scores, times=[per_bin * s for s in bins], A=A, F=F, cum=cum,
                            attn=r["attn"]))
        return out
