"""SeamlessStreaming monotonic text decoder on the CUDA kernels (SURVEY 8a a17).

Reference: models/monotonic_decoder/{model.py:23, monotonic_decoder.py:66-98, monotonic_decoder_layer.py:108-201,
p_choose.py:120-148}; architecture `dense_1b` (builder.py:88-103).  The decoder layers are the NLLB layers of
`UnitYEngine`; each additionally evaluates its PChooseLayer on the cross-attention LayerNorm output.

The forward is the full-prefix (no state bag) one, numerically what the reference's incremental forward computes; the
greedy READ/WRITE policy of `MMATextDecoderAgent` (streaming/agents/online_text_decoder.py:205-387) runs on top of it.
State reuse: everything that depends only on the SOURCE - the pooled encoder output, the four-layer key-energy MLP of every
layer and the cross-attention K/V of every layer (24 x (k/v GEMM + 4 energy GEMMs) per call in round 1) - is computed
once per encoder output and reused by every token of a policy call and by every later call on the same source
(`_source_state`); only the (short) target prefix is recomputed per token."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from ... import _lib, config as cfgmod, ops, synthetic
from ..._lib import check
from ...engine import I32, UnitYEngine
from ...ops import ACT_RELU, F16, Seq


class MonotonicDecoderModel:
    def __init__(self, cfg, state_dict: Dict[str, torch.Tensor], tokenizers, device="cuda", energy_layers: int = 4,
                 temperature: float = 0.2, pre_decision_ratio: int = 2):
        # the shared decoder weights are packed by UnitYEngine (a monotonic checkpoint has no speech encoder: the engine
        # packs the text decoder only)
        self.engine = UnitYEngine(cfg, {k: v for k, v in state_dict.items() if "p_choose_layer" not in k}, tokenizers, device=device)
        self._src_key, self._src = None, None
        self.cfg, self.device = cfg, torch.device(device)
        self.temperature, self.ratio, self.n_energy = temperature, pre_decision_ratio, energy_layers
        self.pw: Dict[str, torch.Tensor] = {}
        self.energy_bias: List[float] = []
        for i in range(cfg.dec_layers):
            p = f"text_decoder.layers.{i}.p_choose_layer"
            for br in ("q_energy_proj", "k_energy_proj"):
                for l in range(energy_layers):
                    n = f"{p}.{br}.layers.{2 * l}"
                    self.pw[n + ".w"] = state_dict[n + ".weight"].to(self.device, F16).contiguous()
                    self.pw[n + ".b"] = state_dict[n + ".bias"].to(self.device, torch.float32).contiguous()
            eb = state_dict.get(p + ".energy_bias")
            self.energy_bias.append(float(eb[0]) if eb is not None else 0.0)

    def _energy(self, x: Seq, prefix: str) -> Seq:
        for l in range(self.n_energy):
            n = f"{prefix}.layers.{2 * l}"
            x = ops.gemm(x, self.pw[n + ".w"], self.cfg.model_dim, self.pw[n + ".b"], act=ACT_RELU)
        return x

    @torch.inference_mode()
    def decode(self, seqs: torch.Tensor, encoder_output: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """seqs (1, L) int64 prefix, encoder_output (1, S, M) fp16 -> (decoder output (1, L, M) fp16,
        p_choose (layers, heads, L, ceil(S/ratio)) fp32)  [monotonic_decoder.py:66-98]."""
        lib = _lib.load()
        eng, c = self.engine, self.cfg
        M, H = c.model_dim, c.num_heads
        assert seqs.shape[0] == 1 and encoder_output.shape[0] == 1, "the streaming decoder runs one stream at a time"
        L, S = seqs.shape[1], encoder_output.shape[1]
        Sp = (S + self.ratio - 1) // self.ratio
        src = self._source_state(encoder_output)
        x = Seq(1, L, M, buf=ops.embed_seq(seqs.to(self.device, I32).contiguous(), eng.w["text_embed"], eng.pos, math.sqrt(M), M))
        p_all = torch.empty((c.dec_layers, H, L, Sp), dtype=torch.float32, device=self.device)
        for i in range(c.dec_layers):
            p = f"text_decoder.layers.{i}"
            x = eng._mha_self(eng._ln(x, p + ".self_attn_layer_norm"), p + ".self_attn", x, causal=True)
            h = eng._ln(x, p + ".encoder_decoder_attn_layer_norm")
            # PChooseLayer on the normalised decoder states and the pooled encoder output
            qe = self._energy(h, p + ".p_choose_layer.q_energy_proj")
            ke = src["ke"][i]
            check(lib.sb_pchoose(qe.buf.data_ptr(), ke.buf.data_ptr(), p_all[i].data_ptr(), L, Sp, H, self.energy_bias[i],
                                 self.temperature, ops._stream()), "sb_pchoose")
            q = eng._lin(h, p + ".encoder_decoder_attn.q_proj", M)
            kv = src["kv"][i]
            att = Seq(1, L, M)
            ops.attention(q.buf, kv[:, :M], kv[:, M:], att.buf, 1, H, L, S, L, 0, S, 0, None)
            x = eng._lin(att, p + ".encoder_decoder_attn.output_proj", M, res1=x)
            x = eng._ffn(eng._ln(x, p + ".ffn_layer_norm"), p + ".ffn", c.dec_ffn_dim, ACT_RELU, x)
        out = eng._ln(x, "text_decoder.layer_norm")
        return out.buf.view(1, L, M), p_all

    def _source_state(self, encoder_output: torch.Tensor):
        """Per-source tensors of every layer: cross-attention K|V and the key-energy projections of the pooled encoder output.
        Keyed by the identity of the encoder-output tensor object (a reference is kept, so the id cannot be recycled): every
        decoder run of a policy call, and the calls that follow a WRITE, pass the same object; a grown source is a new one."""
        key = encoder_output
        if self._src_key is key:
            return self._src
        lib = _lib.load()
        eng, c = self.engine, self.cfg
        M, S = c.model_dim, encoder_output.shape[1]
        Sp = (S + self.ratio - 1) // self.ratio
        enc = Seq(1, S, M, buf=encoder_output.to(self.device, F16).contiguous().view(S, M))
        pooled = Seq(1, Sp, M)
        check(lib.sb_avgpool_time(enc.buf.data_ptr(), pooled.buf.data_ptr(), 1, S, M, self.ratio, ops._stream()), "sb_avgpool_time")
        kv, ke = [], []
        for i in range(c.dec_layers):
            p = f"text_decoder.layers.{i}"
            kv.append(eng._lin(enc, p + ".encoder_decoder_attn.kv", 2 * M).buf)
            ke.append(self._energy(pooled, p + ".p_choose_layer.k_energy_proj"))
        self._src_key, self._src = key, dict(kv=kv, ke=ke, enc=enc)
        self.source_state_builds = getattr(self, "source_state_builds", 0) + 1
        return self._src

    # ---------------------------------------------------------------------------------- many streams at once
    def _build_sources(self, encs: List[torch.Tensor]) -> List[dict]:
        """The source state of several encoder outputs (1, S_b, M) in one pass: padded to (B, S_max) with per-row lengths,
        one K|V GEMM and one energy chain per layer for all of them (AvgPool1d per stream, as it has no row lengths).
        Returns each stream's state as views: kv (layers, S_b, 2M), ke (layers, Sp_b, M)."""
        lib = _lib.load()
        eng, c = self.engine, self.cfg
        M, B, r = c.model_dim, len(encs), self.ratio
        S = [int(e.shape[1]) for e in encs]
        Sp = [(n + r - 1) // r for n in S]
        Smax, Spmax = max(S), max(Sp)
        enc = Seq(B, Smax, M, zero=True)
        pooled = Seq(B, Spmax, M, zero=True)
        ev, pv = enc.buf.view(B, Smax, M), pooled.buf.view(B, Spmax, M)
        for b, e in enumerate(encs):
            ev[b, :S[b]].copy_(e[0])
            check(lib.sb_avgpool_time(ev[b].data_ptr(), pv[b].data_ptr(), 1, S[b], M, r, ops._stream()), "sb_avgpool_time")
        kv = torch.empty((c.dec_layers, B, Smax, 2 * M), dtype=F16, device=self.device)
        ke = torch.empty((c.dec_layers, B, Spmax, M), dtype=F16, device=self.device)
        for i in range(c.dec_layers):
            p = f"text_decoder.layers.{i}"
            eng._lin(enc, p + ".encoder_decoder_attn.kv", 2 * M, out=Seq(B, Smax, 2 * M, buf=kv[i].view(B * Smax, 2 * M)))
            x = pooled
            for l in range(self.n_energy):
                n = f"{p}.p_choose_layer.k_energy_proj.layers.{2 * l}"
                out = Seq(B, Spmax, M, buf=ke[i].view(B * Spmax, M)) if l == self.n_energy - 1 else None
                x = ops.gemm(x, self.pw[n + ".w"], M, self.pw[n + ".b"], act=ACT_RELU, out=out)
        self.source_state_builds = getattr(self, "source_state_builds", 0) + B
        return [dict(kv=kv[:, b, :S[b]], ke=ke[:, b, :Sp[b]], S=S[b], Sp=Sp[b], enc=encs[b]) for b in range(B)]

    def _source_batch(self, encs: List[torch.Tensor]) -> dict:
        """Padded per-layer source state of a batch of streams.  A stream's state is built (with every other new one, in
        one pass) only when its encoder-output object is new; a batch is assembled from the streams' states only when the
        set of streams changes (copies, no arithmetic)."""
        cache = getattr(self, "_src_cache", {})
        new = [e for e in dict.fromkeys(encs) if id(e) not in cache or cache[id(e)]["enc"] is not e]
        if new:
            # new sources start a new tick: the states of sources this batch does not use are never asked for again
            cache = {id(e): cache[id(e)] for e in encs if id(e) in cache and cache[id(e)]["enc"] is e}
            for st in self._build_sources(new):
                cache[id(st["enc"])] = st
            self._src_cache = cache
        key = tuple(id(e) for e in encs)
        bat = getattr(self, "_src_bat", None)
        if bat is not None and bat["key"] == key and all(a is b for a, b in zip(bat["encs"], encs)):
            return bat
        c, M, dev = self.cfg, self.cfg.model_dim, self.device
        sts = [cache[k] for k in key]
        B, Smax, Spmax = len(sts), max(st["S"] for st in sts), max(st["Sp"] for st in sts)
        kv = torch.zeros((c.dec_layers, B, Smax, 2 * M), dtype=F16, device=dev)
        ke = torch.zeros((c.dec_layers, B, Spmax, M), dtype=F16, device=dev)
        for b, st in enumerate(sts):
            kv[:, b, :st["S"]].copy_(st["kv"])
            ke[:, b, :st["Sp"]].copy_(st["ke"])
        lens, = self._upload(torch.tensor([[st["S"] for st in sts], [st["Sp"] for st in sts]], dtype=I32))
        self._src_bat = bat = dict(key=key, encs=list(encs), kv=kv, ke=ke, S=lens[0], Sp=lens[1], Smax=Smax, Spmax=Spmax)
        return bat

    def _upload(self, *parts: torch.Tensor) -> List[torch.Tensor]:
        """int32 host tensors -> device tensors of the same shapes, through one pinned buffer and one asynchronous copy: no
        host sync (a pageable copy would drain the stream).  The caching host allocator does not hand the pinned block out
        again before the copy has run."""
        sizes = [t.numel() for t in parts]
        host = torch.empty(sum(sizes), dtype=I32, pin_memory=True)
        torch.cat([t.reshape(-1) for t in parts], out=host)
        dev = host.to(self.device, non_blocking=True)
        return [v.view(t.shape) for v, t in zip(dev.split(sizes), parts)]

    def _forward(self, seqs: List[List[int]], encoder_outputs: List[torch.Tensor], extra: Optional[torch.Tensor] = None):
        """forward_batch; `extra` (int32 host tensor) goes to the device in the same copy as the token ids and is returned
        as the last element."""
        eng, c = self.engine, self.cfg
        M, H, B = c.model_dim, c.num_heads, len(seqs)
        assert B == len(encoder_outputs) and B > 0 and all(len(t) > 0 for t in seqs)
        src = self._source_batch(encoder_outputs)
        lens = [len(t) for t in seqs]
        L = max(lens)
        ids = torch.full((B, L), c.text_eos, dtype=I32)
        for b, t in enumerate(seqs):
            ids[b, :lens[b]] = torch.tensor(t, dtype=I32)
        parts = [ids, torch.tensor(lens, dtype=I32)] + ([extra] if extra is not None else [])
        ids, q_lens, *extra_dev = self._upload(*parts)
        x = Seq(B, L, M, buf=ops.embed_seq(ids, eng.w["text_embed"], eng.pos, math.sqrt(M), M))
        p_last = torch.empty((c.dec_layers, B, H), dtype=torch.float32, device=self.device)
        Smax, Spmax = src["Smax"], src["Spmax"]
        for i in range(c.dec_layers):
            p = f"text_decoder.layers.{i}"
            x = eng._mha_self(eng._ln(x, p + ".self_attn_layer_norm"), p + ".self_attn", x, causal=True)
            h = eng._ln(x, p + ".encoder_decoder_attn_layer_norm")
            qe = self._energy(h, p + ".p_choose_layer.q_energy_proj")
            ke = Seq(B, Spmax, M, buf=src["ke"][i].view(B * Spmax, M))
            ops.pchoose_ragged(qe, ke, q_lens, src["Sp"], H, self.energy_bias[i], self.temperature, p_last[i])
            q = eng._lin(h, p + ".encoder_decoder_attn.q_proj", M)
            kv = src["kv"][i].view(B * Smax, 2 * M)
            att = Seq(B, L, M)
            ops.attention(q.buf, kv[:, :M], kv[:, M:], att.buf, B, H, L, Smax, L, 0, Smax, 0, src["S"])
            x = eng._lin(att, p + ".encoder_decoder_attn.output_proj", M, res1=x)
            x = eng._ffn(eng._ln(x, p + ".ffn_layer_norm"), p + ".ffn", c.dec_ffn_dim, ACT_RELU, x)
        out = eng._ln(x, "text_decoder.layer_norm")
        return out, p_last, q_lens, (extra_dev[0] if extra_dev else None)

    @torch.inference_mode()
    def forward_batch(self, seqs: List[List[int]], encoder_outputs: List[torch.Tensor]):
        """The decoder over a batch of streams: token prefixes of different lengths, each with its own encoder output
        (1, S_b, M) fp16.  Runs the layers once over the padded prefixes (causal self-attention needs no lengths: a row
        never attends past itself; cross-attention masks each stream's source by its length).  Returns (decoder output
        Seq (B, L_max, M), p_last (layers, B, heads) fp32: p_choose of each stream's newest position against its last
        pooled source position, target lengths int32 (B,) on the device).  No host sync."""
        return self._forward(seqs, encoder_outputs)[:3]

    def _newest_rows(self, out: Seq, q_lens: torch.Tensor) -> torch.Tensor:
        rows = torch.arange(out.B, device=self.device, dtype=I32) * out.T + q_lens - 1
        return out.buf.index_select(0, rows)

    @torch.inference_mode()
    def decode_batch(self, seqs: List[List[int]], encoder_outputs: List[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """forward_batch reduced to what the policy reads: (newest-position decoder output (B, M) fp16, the input of the
        vocabulary projection; p_last (layers, B, heads) fp32)."""
        out, p_last, q_lens, _ = self._forward(seqs, encoder_outputs)
        return self._newest_rows(out, q_lens), p_last

    @torch.inference_mode()
    def policy_round(self, seqs: List[List[int]], encoder_outputs: List[torch.Tensor], ctl: List[List[int]]) -> torch.Tensor:
        """One decoder run of every stream still inside a policy call: decode_batch, the vocabulary projection of the newest
        positions and sb_policy_decide.  ctl: one ops.policy_ctl row per stream, uploaded with the token ids in one
        asynchronous copy.  Returns (B, 2) int32 on the device, {token, float bits of the decision value} per stream, for the
        caller to read once: the round makes no host sync of its own."""
        out, p_last, q_lens, ctl_dev = self._forward(seqs, encoder_outputs, torch.tensor(ctl, dtype=I32))
        logits = self.project(self._newest_rows(out, q_lens)[:, None])[:, 0]
        return ops.policy_decide(logits, ctl_dev, p_last)

    def project(self, decoder_output: torch.Tensor) -> torch.Tensor:
        B, L, M = decoder_output.shape
        return ops.gemm_raw(decoder_output.contiguous().view(B * L, M), self.engine.w["text_embed"], self.cfg.text_vocab,
                            out_f32=True).view(B, L, -1)[:, :, :self.cfg.text_vocab]


def load_monotonic_decoder_model(arch: str = "base_v2", device="cuda", state_dict=None, tokenizers=None, seed: int = 2) -> MonotonicDecoderModel:
    cfg = cfgmod.UNITY_ARCHS[cfgmod.MODEL_CARDS.get(arch, arch)]()
    if state_dict is None:
        state_dict = synthetic.make_monotonic_state_dict(cfg, seed=seed)
    if tokenizers is None:
        tokenizers = synthetic.make_tokenizers(cfg)
    return MonotonicDecoderModel(cfg, state_dict, tokenizers, device=device)
