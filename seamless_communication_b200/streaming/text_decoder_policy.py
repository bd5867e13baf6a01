"""EMMA READ/WRITE policy of the streaming text decoder: behavioural mirror of `MMATextDecoderAgent.policy`,
`run_decoder`, `get_blocked_ngrams` and `maybe_block_ngrams` (reference
streaming/agents/online_text_decoder.py:205-243, 260-387), pinned call by call against the reference agent by
tests/golden/policy_traces.json.  SimulEval is not available offline, so this is a plain class: feed it the encoder
output accumulated so far, get back the newly written token ids."""
from __future__ import annotations

from typing import List, Optional, Sequence, Set, Tuple

import torch


class MMATextDecoderPolicy:
    """Arguments carry the reference's CLI defaults (online_text_decoder.py:96-185)."""

    def __init__(self, model, tgt_lang: Optional[str] = None, decision_threshold: float = 0.5, decision_method: str = "min",
                 p_choose_start_layer: int = 0, max_len_a: int = 1, max_len_b: int = 200, max_consecutive_writes: int = 50,
                 min_starting_wait: int = 1, no_early_stop: bool = False, block_ngrams: bool = False,
                 prefix: Optional[Sequence[int]] = None, eos_idx: Optional[int] = None):
        self.model = model
        if prefix is None:  # [</s>, __lang__]: the "target" mode prefix of the NLLB tokenizer (:83-87, 135-140)
            prefix = [model.cfg.text_eos, model.engine.text_tokenizer.lang_index(tgt_lang)]
        self.prefix = list(prefix)
        self.eos = model.cfg.text_eos if eos_idx is None else eos_idx
        if decision_method not in ("min", "mean", "median"):
            raise ValueError(f"`decision_method` must be 'min', 'mean' or 'median', but is '{decision_method}' instead.")
        self.threshold, self.method, self.start_layer = decision_threshold, decision_method, p_choose_start_layer
        self.max_len_a, self.max_len_b, self.max_writes = max_len_a, max_len_b, max_consecutive_writes
        self.min_starting_wait, self.no_early_stop, self.block_ngrams = min_starting_wait, no_early_stop, block_ngrams
        self.reset()

    def reset(self) -> None:  # DecoderAgentStates.reset (:27-32)
        self.target_indices: List[int] = []
        self.target_finished = False
        self.ngram_block_count = 0
        self._call = None

    def _decide(self, p_choose: torch.Tensor) -> float:
        last = p_choose[self.start_layer:, :, -1, -1]  # (layers, heads) (:233-243)
        if self.method == "min":
            return float(last.min())
        if self.method == "mean":
            return float(last.mean())
        return float(last.median())

    def _run_decoder(self, encoder_output, pred: List[int]) -> Tuple[int, float]:
        """run_decoder (:205-243).  The reference feeds only the newest token and keeps an IncrementalStateBag per policy
        call; this engine re-runs the (short) prefix, which yields the same last-position outputs."""
        ids = torch.tensor([self.prefix + self.target_indices + pred], dtype=torch.int64)
        dec, p_choose = self.model.decode(ids, encoder_output)
        logits = self.model.project(dec[:, -1:])[0, -1].float().clone()
        blocked = self.blocked_ids()
        if blocked:
            logits[blocked] = float("-inf")
        return int(logits.argmax().item()), self._decide(p_choose)

    def _blocked_ngrams(self) -> Optional[Set[str]]:  # get_blocked_ngrams (:260-274)
        if not self.block_ngrams:
            return None
        t, out = self.target_indices, set()
        if len(t) >= 4:
            out.update((str(t[-4:]), str(t[-4:-2]), str(t[-4:-1])))
        if len(t) >= 3:
            out.update((str(t[-3:]), str(t[-3:-1])))
        if len(t) >= 2:
            out.add(str(t[-2:]))
        return out

    def _maybe_block(self, pred: List[int], blocked: Optional[Set[str]], index: int, source_finished: bool) -> bool:
        """maybe_block_ngrams (:276-302): forces a READ when an n-gram repeats before the source is finished; trims the
        tokens that started the repeat from `pred` in place."""
        if not self.block_ngrams or source_finished:
            return False
        assert blocked is not None
        all_indices = self.target_indices + pred + [index]
        for n in (3, 2):
            if len(all_indices) >= n and self.ngram_block_count <= 4:
                if str(all_indices[-n:]) in blocked:
                    self.ngram_block_count += 1
                    pred[:] = pred[: -(n - 1)]
                    return True
                blocked.add(str(all_indices[-n:]))
        return False

    # -------------------------------------------------------------------------- one policy call, a token at a time
    # policy() below is begin() followed by decoder runs fed to step() until it returns.  A multi-stream driver
    # (StreamingS2STBatch) calls the same three methods, so that every stream takes exactly the decisions policy() takes,
    # while the decoder runs of many streams go through the device as one batch.
    def begin(self, source_len: int, source_finished: bool) -> Optional[Tuple[List[int], bool]]:
        """Starts one policy call on `source_len` encoder frames.  Returns the call's result when it ends without running
        the decoder; otherwise None, and the call continues with step()."""
        self._call = None
        if source_len == 0:
            return [], False
        if source_len < self.min_starting_wait and not source_finished:
            return [], False
        if self.target_finished:
            return [], True
        self._call = dict(max_len=self.max_len_a * source_len + self.max_len_b, pred=[], finished=False,
                          blocked=self._blocked_ngrams(), source_finished=source_finished)
        return None

    @property
    def pending(self) -> List[int]:
        """Tokens written so far by the current call (not yet in target_indices)."""
        return self._call["pred"]

    def decoder_ids(self) -> List[int]:
        """The token prefix of the current call's next decoder run."""
        return self.prefix + self.target_indices + self._call["pred"]

    def blocked_ids(self) -> List[int]:
        """Token ids set to -inf before the argmax of the current call's next decoder run (the `block_ngrams and
        source_finished` rule of run_decoder, at most 4)."""
        if self.block_ngrams and self._call["source_finished"]:
            return (self.target_indices + self._call["pred"])[-4:]
        return []

    def step(self, index: int, prob: float) -> Optional[Tuple[List[int], bool]]:
        """Feeds the newest position's token and decision value of one decoder run (:344-369).  Returns the call's result
        (as policy() does) when the call ends, or None when it wants another decoder run."""
        c = self._call
        pred, max_len, source_finished = c["pred"], c["max_len"], c["source_finished"]
        if self.no_early_stop and not source_finished and (prob < self.threshold or index == self.eos):
            if prob == 1.0:
                c["pred"] = pred = []
            return self._end()
        if self._maybe_block(pred, c["blocked"], index, source_finished):
            return self._end()
        if c["finished"] or index == self.eos or len(self.target_indices) + len(pred) > max_len:
            c["finished"] = True
            return self._end()
        if prob < self.threshold and not source_finished:
            return self._end()  # READ
        if len(self.target_indices) + len(pred) >= max_len or len(pred) >= self.max_writes:
            return self._end()
        pred.append(index)
        return None

    def _end(self) -> Tuple[List[int], bool]:
        c, self._call = self._call, None
        pred, finished = c["pred"], c["finished"]
        self.target_indices += pred
        if len(pred) > 0 or finished:
            # the reference re-checks the budget with `states.target_indices + pred_indices` AFTER the append above, i.e.
            # it counts this call's tokens twice (:374-377); mirrored
            finished = finished or len(self.target_indices) + len(pred) > c["max_len"]
            self.ngram_block_count = 0
            self.target_finished = finished
            return pred, finished
        return [], False

    @torch.inference_mode()
    def policy(self, encoder_output: torch.Tensor, source_finished: bool) -> Tuple[List[int], bool]:
        """One call of the agent's policy (:304-387).  Returns (tokens written by this call, finished); ([], False) is a
        READ.  As under SimulEval, call again with the same source after a WRITE; feed more source after a READ."""
        source_len = 0 if encoder_output is None else int(encoder_output.shape[1])
        done = self.begin(source_len, source_finished)
        while done is None:
            index, prob = self._run_decoder(encoder_output, self.pending)
            done = self.step(index, prob)
        return done
