"""CPU oracle of the beam search with fairseq2's NGramRepeatBlockProcessor (the step processor of the reference CLI's
`--text_generation_ngram_blocking` / `--unit_generation_ngram_blocking`), test infrastructure like
oracle/unity_oracle.py.  This subclass adds the processor and leaves the pinned search of `UnityOracle.beam_search`
untouched; without a processor its `beam_search` is the same search step for step.  It serves the text decoder and,
over the renamed AR T2U weights (tests/test_v1_s2st.py::unit_oracle), the unit decoder.

fairseq2 is not in the tree, so the processor's semantics are recalled [fs2-recall] (DESIGN.md section 15):
  * `NGramRepeatBlockProcessor(ngram_size)` raises ValueError for a size below 1;
  * it runs where BannedSequenceProcessor runs (tests/oracle_mintox.py): at every selecting step (step >= P-1), never in
    the prompt bootstrap, on the log-probabilities after log_softmax and after the _tweak_lprobs tweaks, the forced-EOS
    step included;
  * it sees seqs[row, :step+1]: the row's whole hypothesis, the forced prompt tokens [</s>, __lang__] included;
  * every start i with i + n - 1 <= step whose n-1 tokens equal the row's last n-1 tokens bans the token at i + n - 1
    (overlapping occurrences count); a row of fewer than n tokens has no start and bans nothing, so the first step that
    can ban is step = n-1, with the single start i = 0;
  * n == 1 bans every token the row holds.  The prompt's </s> is EOS, so no hypothesis can finish;
  * a banned token's lprob becomes -inf; the normaliser is taken before, so every other lprob is kept bit for bit.
"""
from __future__ import annotations

import math
import os
import sys
from typing import List, Tuple

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle.unity_oracle import UnityOracle, key_mask  # noqa: E402


def ngram_bans(hist: List[int], n: int) -> List[int]:
    """NGramRepeatBlockProcessor(n) on one row holding `hist` (seqs[row, :step+1]): the token after each earlier
    occurrence of the row's last n-1 tokens, one entry per start."""
    last = hist[len(hist) - (n - 1):]
    return [hist[i + n - 1] for i in range(len(hist) - n + 1) if hist[i:i + n - 1] == last]


def repeated_ngrams(ids: List[int], n: int) -> List[Tuple[int, ...]]:
    """The n-grams that occur more than once in `ids` (overlaps count)."""
    seen, out = set(), []
    for i in range(len(ids) - n + 1):
        g = tuple(ids[i:i + n])
        if g in seen:
            out.append(g)
        seen.add(g)
    return out


class UnityOracleNGram(UnityOracle):
    def beam_search(self, enc, enc_lens, prefix: List[int], beam=5, soft_max=(1, 200), hard_max=1024,
                    len_penalty=1.0, unk_penalty=0.0, min_seq_len=1, trace=None, ngram=None):
        """UnityOracle.beam_search (BeamSearchSeq2SeqGenerator as mirrored in fairseq2.cpp:1097-1608) with n-gram repeat
        blocking of size `ngram` applied after the tweaks.  Returns per sentence the finished hypotheses [(score, ids)],
        best first."""
        V = self.c["text_vocab"]
        eos, pad, unk = self.c["text_eos"], self.c["text_pad"], self.c["text_unk"]
        results = []
        for n in range(enc.shape[0]):
            S_enc = int(enc_lens[n]) if enc_lens is not None else enc.shape[1]
            src_len = enc.shape[1]
            a, b = soft_max
            max_len = hard_max if a <= 0 else min(hard_max, int(a * src_len) + b)
            e = enc[n:n + 1].expand(beam, -1, -1)
            ekm = key_mask(torch.full((beam,), S_enc), enc.shape[1]) if enc_lens is not None else None
            caches = [({}, {"static": True}) for _ in range(self.c["dec_layers"])]
            seqs = torch.zeros(beam, max_len, dtype=torch.long)
            scores = torch.zeros(beam, max_len)
            P = len(prefix)
            seqs[:, :P] = torch.tensor(prefix)
            if P > 1:  # bootstrap: feed prefix[:-1], score prefix[1:] (no processor)
                h = self.decoder(self.embed_text(seqs[:, :P - 1], 0), e, ekm, caches)
                lp = torch.log_softmax(self.project(h).float(), dim=-1)
                acc = 0.0
                for i in range(1, P):
                    acc = acc + float(lp[0, i - 1, prefix[i]])
                    scores[:, i] = acc
                if trace is not None and n == trace.get("sentence", 0):
                    trace["prefix_scores"] = scores[0, :P].clone()
            finished: List[Tuple[float, List[int]]] = []
            done = False
            for step in range(P - 1, max_len - 1):
                h = self.decoder(self.embed_text(seqs[:, step:step + 1], step), e, ekm, caches)
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
                if ngram:
                    for row in range(beam):
                        lp[row, ngram_bans(seqs[row, :step + 1].tolist(), ngram)] = -math.inf
                if step == P - 1:  # first step: beam 0 only
                    cand = lp[0:1] + scores[0:1, step:step + 1]
                else:
                    cand = lp + scores[:, step:step + 1]
                top_s, top_i = torch.topk(cand.reshape(-1), min(2 * beam, V - 1))
                bi, ti, si = [], [], []
                for c_s, c_i in zip(top_s.tolist(), top_i.tolist()):
                    bm, tok = c_i // V, c_i % V
                    if tok == eos and c_s != -math.inf:
                        finished.append((c_s / float((step + 1) ** len_penalty), seqs[bm, :step + 1].tolist() + [tok]))
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
                seqs, scores = seqs[bidx].clone(), scores[bidx].clone()
                seqs[:, step + 1] = torch.tensor(ti)
                scores[:, step + 1] = torch.tensor(si)
                for sc, _ in caches:
                    sc["k"], sc["v"] = sc["k"][bidx], sc["v"][bidx]
                if trace is not None and n == trace.get("sentence", 0):
                    trace.setdefault("beam_idx", []).append(bidx.clone())
            order = sorted(range(len(finished)), key=lambda j: -finished[j][0])
            if trace is not None and n == trace.get("sentence", 0):
                trace["finished"] = list(finished)
                trace["max_len"] = max_len
            results.append([finished[j] for j in order])
        return results
