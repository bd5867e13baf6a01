"""SeamlessStreaming S2ST for many concurrent streams.  Every stream computes exactly what `StreamingS2ST` computes for it
alone; what is shared is the device work of a tick:

    policy   the WRITE loop of every stream inside a policy call advances one token per round: one batched decoder run
             over all of their padded prefixes (MonotonicDecoderModel.policy_round), one sb_policy_decide and ONE host read
             of (token, decision value) for all streams, instead of a batch-1 decoder run and two host reads per token
    features the decoder features of every stream that wrote in the tick, in one batched decoder run

Each stream keeps its own feature extractor, encoder frames, policy state, NAR T2U state, options and target language.
The speech encoder, the NAR T2U and the vocoder run per stream (DESIGN.md, "Many streams"): the encoder's adaptor reads
frames past a row's length, so a padded batch is not the stream alone."""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Tuple

import numpy as np
import torch

from .. import ops
from .pipeline import NARUnitDecoder, OfflineW2vBertEncoder, OnlineFeatureExtractor
from .text_decoder_policy import MMATextDecoderPolicy


class _Stream:
    __slots__ = ("sid", "tgt_lang", "features", "encoder", "policy", "units", "enc_out", "text_ids", "new_ids", "done",
                 "finished")


class StreamingS2STBatch:
    def __init__(self, unity_model, monotonic_model, vocoder, source_segment_ms: int = 320):
        self.unity, self.mono, self.vocoder = unity_model, monotonic_model, vocoder
        self.device = torch.device(monotonic_model.device)
        self.segment_samples = int(source_segment_ms * 16)
        self.comma = monotonic_model.engine.text_tokenizer.model.token_to_index(",")
        self.streams: Dict[int, _Stream] = {}
        self._next_id = 0
        self.latencies_ms: List[float] = []  # device time of every push (CUDA events)
        self.rounds = 0       # policy rounds run
        self.host_reads = 0   # device-to-host reads of the policy's decisions (one per round)

    def _make_features(self):
        return OnlineFeatureExtractor(self.unity.engine.device)

    def add_stream(self, tgt_lang: str, min_starting_wait_w2vbert: Optional[int] = 192, decision_threshold: float = 0.5,
                   no_early_stop: bool = True, max_len_a: int = 0, max_len_b: int = 100, min_unit_chunk_size: int = 50,
                   d_factor: float = 1.0, **policy_kw) -> int:
        """A new stream with StreamingS2ST's options and defaults; returns its id."""
        s = _Stream()
        s.sid, s.tgt_lang = self._next_id, tgt_lang
        self._next_id += 1
        s.features = self._make_features()
        s.encoder = OfflineW2vBertEncoder(self.unity, min_starting_wait_w2vbert)
        s.policy = MMATextDecoderPolicy(self.mono, tgt_lang=tgt_lang, decision_threshold=decision_threshold,
                                        no_early_stop=no_early_stop, max_len_a=max_len_a, max_len_b=max_len_b, **policy_kw)
        s.units = NARUnitDecoder(self.unity, min_unit_chunk_size, d_factor)
        s.enc_out, s.text_ids, s.new_ids, s.done, s.finished = None, [], [], False, False
        self.streams[s.sid] = s
        return s.sid

    def close(self, sid: int) -> None:
        """Forgets a stream; its id is not reused."""
        del self.streams[sid]

    def text_ids(self, sid: int) -> List[int]:
        return self.streams[sid].text_ids

    # ---------------------------------------------------------------------------------------------- one tick
    @torch.inference_mode()
    def push(self, samples: Dict[int, torch.Tensor], finished: Iterable[int] = ()) -> Dict[int, Tuple[List[int], Optional[torch.Tensor], Optional[torch.Tensor]]]:
        """One source segment for each stream in `samples` (streams in `finished` receive their last one; they may have no
        samples).  Returns, for each of these streams, what StreamingS2ST.push returns: (new text ids, new units | None,
        new waveform | None)."""
        finished = set(finished)
        unknown = (set(samples) | finished) - set(self.streams)
        if unknown:
            raise KeyError(f"unknown stream ids {sorted(unknown)}")
        timing = self.device.type == "cuda"
        if timing:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        ids = sorted(set(samples) | finished)
        calls: List[_Stream] = []
        for sid in ids:
            s = self.streams[sid]
            s.finished = sid in finished
            s.new_ids, s.done = [], False
            x = samples.get(sid)
            fb = s.features.push(x if x is not None else torch.zeros(0))
            enc = s.encoder.push(fb, s.finished)
            if enc is not None:
                s.enc_out = enc
            if s.enc_out is not None and (enc is not None or s.finished):
                calls.append(s)
        self._policy(calls)
        units, wavs = self._emit([s for s in calls if s.new_ids or s.done])
        out = {}
        for sid in ids:
            s = self.streams[sid]
            s.text_ids += s.new_ids
            out[sid] = (s.new_ids, units.get(sid), wavs.get(sid))
        if timing:
            e1.record()
            torch.cuda.synchronize()
            self.latencies_ms.append(e0.elapsed_time(e1))
        return out

    def _after_call(self, s: _Stream, result) -> bool:
        """A policy call of s ended with `result`; as under SimulEval, a WRITE that did not finish asks again on the same
        source.  Returns True while s needs decoder runs."""
        while result is not None:
            pred, s.done = result
            s.new_ids += pred
            if not pred or s.done:
                return False
            result = s.policy.begin(int(s.enc_out.shape[1]), s.finished)
        return True

    def _policy(self, calls: List[_Stream]) -> None:
        """The policy calls of a tick, one round per token position; a round makes exactly one host sync, the read of its
        decisions."""
        layers = self.mono.cfg.dec_layers
        active = [s for s in calls if self._after_call(s, s.policy.begin(int(s.enc_out.shape[1]), s.finished))]
        while active:
            seqs = [s.policy.decoder_ids() for s in active]
            ctl = [ops.policy_ctl(s.policy.blocked_ids(), s.policy.method, s.policy.start_layer, layers) for s in active]
            dec = self.mono.policy_round(seqs, [s.enc_out for s in active], ctl).cpu()  # the round's one host read
            self.rounds += 1
            self.host_reads += 1
            tok = dec[:, 0].tolist()
            if min(tok) < 0:
                raise RuntimeError("sb_policy_decide refused a stream's options")
            prob = dec[:, 1].numpy().view(np.float32).tolist()
            active = [s for s, t, p in zip(active, tok, prob) if self._after_call(s, s.policy.step(t, p))]

    def _emit(self, streams: List[_Stream]):
        """UnitYMMATextDecoderAgent.postprocess + NAR T2U + vocoder (StreamingS2ST.push) for the streams that wrote or
        finished: the decoder features in one batched run, then units and waveform per stream."""
        units, wavs = {}, {}
        if not streams:
            return units, wavs
        eos = self.mono.cfg.text_eos
        lists = []
        for s in streams:
            t = s.policy.prefix + s.policy.target_indices
            if s.new_ids and s.new_ids[-1] != eos:
                t = t + [self.comma]
            lists.append(t)
        out, _, _ = self.mono.forward_batch(lists, [s.enc_out for s in streams])
        feats = out.buf.view(out.B, out.T, out.C)
        for b, (s, t) in enumerate(zip(streams, lists)):
            u, _ = s.units.push(feats[b:b + 1, :len(t)], t, s.done)
            if u is not None:
                units[s.sid] = u
                if u.numel() > 0:
                    wavs[s.sid] = self.vocoder(u[None], s.tgt_lang, -1, dur_prediction=False)[0, 0]
        return units, wavs
