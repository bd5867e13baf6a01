"""SeamlessStreaming for many concurrent streams (streaming/batch.py): the token-at-a-time policy interface against the
reference agent's traces, the multi-stream driver's bookkeeping with a stub model (CPU), the two policy kernels against
sb_pchoose and a float64 restatement, and whole streams against StreamingS2ST run alone (GPU)."""
import importlib.util
import json
import math
import os
import re
import warnings

import numpy as np
import pytest
import torch

from seamless_communication_b200 import _lib, config as C, ops as O, synthetic as S
from seamless_communication_b200.ops import Seq
from seamless_communication_b200.streaming import MMATextDecoderPolicy, StreamingS2STBatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
dev = "cuda"


def _script():
    spec = importlib.util.spec_from_file_location("policy_script", os.path.join(G, "policy_script.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _host_decision(ps, ids, src, salt, blocked, method, layer0):
    """What the single-stream policy computes from the scripted decoder run: masked argmax and the p_choose reduction."""
    logits, probs = ps.script(ids, src, salt)
    lg = torch.from_numpy(logits).float()
    if blocked:
        lg[blocked] = float("-inf")
    last = torch.from_numpy(probs)[layer0:]
    prob = {"min": last.min(), "mean": last.mean(), "median": last.median()}[method]
    return int(lg.argmax()), float(prob)


# ------------------------------------------------------------------------------------------------ CPU
def test_token_at_a_time_policy_reproduces_reference_traces():
    """begin / decoder_ids / blocked_ids / step, driven the way StreamingS2STBatch drives them, reproduce every golden
    scenario of the reference agent call by call."""
    ps = _script()
    traces = json.load(open(os.path.join(G, "policy_traces.json")))
    assert set(traces) == {s["name"] for s in ps.SCENARIOS}
    for name, tr in traces.items():
        a = tr["args"]
        pol = MMATextDecoderPolicy(None, prefix=[ps.EOS, 5], eos_idx=ps.EOS, decision_threshold=a["decision_threshold"],
                                   decision_method=a["decision_method"], p_choose_start_layer=a["p_choose_start_layer"],
                                   max_len_a=a["max_len_a"], max_len_b=a["max_len_b"],
                                   max_consecutive_writes=a["max_consecutive_write"], min_starting_wait=a["min_starting_wait"],
                                   no_early_stop=a["no_early_stop"], block_ngrams=a["block_ngrams"])
        for i, call in enumerate(tr["calls"]):
            res = pol.begin(call["src"], call["final"])
            while res is None:
                tok, prob = _host_decision(ps, pol.decoder_ids(), call["src"], tr["salt"], pol.blocked_ids(), pol.method,
                                           pol.start_layer)
                res = pol.step(tok, prob)
            new, finished = res
            if call["action"] == "R":
                assert (new, finished) == ([], False), (name, i, new, finished)
            else:
                assert new == call["tokens"] and finished == call["finished"], (name, i, new, call)
        assert pol.target_finished == tr["calls"][-1].get("finished", False), name


def test_header_declares_and_library_exports_the_policy_kernels():
    hdr = open(os.path.join(ROOT, "include", "seamless_b200.h")).read()
    for name in ("sb_pchoose_ragged", "sb_policy_decide"):
        assert re.search(r"\bint " + name + r"\(", hdr), name
        assert name in _lib.PROTOTYPES and hasattr(_lib.load(), name), name
    consts = dict(re.findall(r"#define (SB_POLICY_\w+) (\d+)", hdr))
    assert {k: int(v) for k, v in consts.items()} == {"SB_POLICY_MIN": 0, "SB_POLICY_MEAN": 1, "SB_POLICY_MEDIAN": 2,
                                                      "SB_POLICY_MAX_BLOCKED": 4, "SB_POLICY_MAX_VALUES": 4096, "SB_POLICY_CTL": 6}
    assert O.POLICY_METHODS == {"min": 0, "mean": 1, "median": 2} and (O.POLICY_MAX_BLOCKED, O.POLICY_CTL) == (4, 6)
    assert O.policy_ctl([7, 9], "median", 1, 24) == [7, 9, -1, -1, 2, 1]


def test_policy_ctl_reads_the_start_layer_as_the_single_stream_slice_does():
    """p_choose[start:] in the single-stream decision: negative starts count from the end and clamp at 0; a start that
    leaves no layer raises there (reduction of an empty tensor), and policy_ctl raises instead of letting the kernel
    return its {-1, NaN} refusal."""
    for start in range(-30, 24):
        assert O.policy_ctl([], "min", start, 24)[5] == range(24)[start:].start
        assert len(range(24)[O.policy_ctl([], "min", start, 24)[5]:]) == len(torch.zeros(24)[start:])
    for bad in (24, 25, 100):
        with pytest.raises(ValueError):
            O.policy_ctl([], "min", bad, 24)
    with pytest.raises(ValueError):
        O.policy_ctl([], "max", 0, 24)
    with pytest.raises(ValueError):
        O.policy_ctl([1, 2, 3, 4, 5], "min", 0, 24)


# ---- a stub model: every stage on the CPU, deterministic in what each stream has received
class _StubEngine:
    M = 4

    def __init__(self):
        self.device = torch.device("cpu")

    def encode_speech(self, x, lens):  # 8 fbank frames per encoder frame; values carry the frame count
        n = int(lens[0])
        S_ = n // 8 + 1
        buf = torch.full((S_, self.M), float(n))
        return Seq(1, S_, self.M, buf=buf), torch.tensor([S_])

    def t2u(self, dseq, ts, duration_factor=1.0):  # two units per token
        L = ts.shape[1]
        units = torch.arange(2 * L)[None]
        return units, torch.tensor([2 * L]), dict(dur=torch.full((1, L), 2))


class _StubUnity:
    def __init__(self):
        self.engine = _StubEngine()
        self.config = type("cfg", (), dict(fbank_stride=2))()


class _StubTok:
    def __init__(self):
        self.model = self

    def token_to_index(self, t):
        return 11

    def lang_index(self, lang):
        return 100 + len(lang)


class _StubMono:
    """policy_round: a token per (stream source length, prefix length); decision value 0.9 until the prefix holds 3
    written tokens per 4 source frames, then 0.1 (READ); EOS (2) after 12 written tokens."""

    def __init__(self):
        self.device = torch.device("cpu")
        self.cfg = type("cfg", (), dict(text_eos=2, dec_layers=3))()
        self.engine = type("eng", (), dict(text_tokenizer=_StubTok(),
                                           device=torch.device("cpu")))()
        self.round_sizes = []

    def policy_round(self, seqs, encs, ctl):
        self.round_sizes.append(len(seqs))
        out = torch.zeros((len(seqs), 2), dtype=torch.int32)
        for b, (t, e) in enumerate(zip(seqs, encs)):
            written, src = len(t) - 2, int(e.shape[1])
            out[b, 0] = 2 if written >= 12 else 20 + (written + src) % 7
            out[b, 1] = int(np.float32(0.9 if written < 3 * src // 4 else 0.1).view(np.int32))
        return out

    def forward_batch(self, seqs, encs):
        L = max(len(t) for t in seqs)
        return Seq(len(seqs), L, 4, buf=torch.zeros(len(seqs) * L, 4)), None, None


class _StubFeatures:
    def push(self, samples):  # one fbank frame per 160 samples, no residual
        k = samples.numel() // 160
        return None if k == 0 else torch.zeros(k, 80)


class _StubBatch(StreamingS2STBatch):
    def _make_features(self):
        return _StubFeatures()


def _stub_driver():
    mono = _StubMono()
    drv = _StubBatch(_StubUnity(), mono, lambda u, lang, spk, dur_prediction: torch.ones(1, 1, u.numel()))
    return drv, mono


def test_driver_bookkeeping_late_start_early_finish_close_and_starting_wait():
    drv, mono = _stub_driver()
    seg = torch.zeros(5120)  # 32 fbank frames, 4 encoder frames per tick
    a = drv.add_stream("spa", min_starting_wait_w2vbert=None, min_unit_chunk_size=1)
    b = drv.add_stream("fra", min_starting_wait_w2vbert=None, min_unit_chunk_size=1)
    c = drv.add_stream("deu", min_starting_wait_w2vbert=64, min_unit_chunk_size=1)  # waits for 64 fbank frames
    out = drv.push({a: seg, c: seg})
    assert set(out) == {a, c}
    assert out[c] == ([], None, None)  # below min_starting_wait: READ, no decoder run
    assert drv.streams[c].enc_out is None
    assert len(out[a][0]) > 0 and out[a][1] is not None and out[a][2] is not None
    assert mono.round_sizes and mono.round_sizes[0] == 1  # only stream a was in the policy
    # b starts late; a finishes early (its final tick carries no samples)
    mono.round_sizes.clear()
    out = drv.push({b: seg, c: seg}, finished={a})
    assert set(out) == {a, b, c}
    assert drv.streams[c].enc_out is not None and drv.rounds == drv.host_reads
    assert max(mono.round_sizes) >= 2  # several streams shared a round
    # close while writing: b has written and is not finished; the others go on unaffected
    assert drv.text_ids(b) and not drv.streams[b].done
    drv.close(b)
    with pytest.raises(KeyError):
        drv.push({b: seg})
    out = drv.push({c: seg}, finished={c})
    assert set(out) == {c} and drv.streams[c].done
    assert drv.rounds == drv.host_reads
    with pytest.raises(KeyError):
        drv.close(b)


def test_driver_streams_match_the_same_stream_driven_alone():
    """Bookkeeping only: with the stub model, each stream's outputs inside a batch equal its outputs in a driver of its own,
    whatever the other streams do and whenever they start."""
    starts, lengths = [0, 1, 3, 0], [5, 3, 2, 1]
    seg = torch.zeros(5120)

    def run(which):
        drv, _ = _stub_driver()
        ids = {i: drv.add_stream("spa", min_starting_wait_w2vbert=None, min_unit_chunk_size=3, max_len_b=9) for i in which}
        got = {i: [] for i in which}
        for t in range(max(s + n for s, n in zip(starts, lengths))):
            live = [i for i in which if starts[i] <= t < starts[i] + lengths[i]]
            if not live:
                continue
            fin = {ids[i] for i in live if t == starts[i] + lengths[i] - 1}
            res = drv.push({ids[i]: seg for i in live}, finished=fin)
            for i in live:
                n, u, w = res[ids[i]]
                got[i].append((n, None if u is None else u.tolist(), None if w is None else w.shape[0]))
        return got

    together = run(range(4))
    for i in range(4):
        assert together[i] == run([i])[i], i


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("heads", [2, 16])
def test_pchoose_ragged_equals_sb_pchoose_per_stream(heads):
    """Each stream's (newest position, last pooled position) value equals sb_pchoose run on that stream alone, bit for bit;
    lengths 1 and past 64, padded layouts whose padding rows are NaN (never read)."""
    lib = _lib.load()
    torch.manual_seed(0)
    Ls, Sps = [1, 5, 70, 33, 2, 64], [1, 80, 3, 65, 1, 17]
    B, D = len(Ls), heads * 64
    Lr, Sr = max(Ls) + 3, max(Sps) + 2
    q = torch.full((B * Lr, D), float("nan"), dtype=torch.float16, device=dev)
    k = torch.full((B * Sr, D), float("nan"), dtype=torch.float16, device=dev)
    for b in range(B):
        q[b * Lr:b * Lr + Ls[b]] = torch.randn(Ls[b], D, device=dev).half()
        k[b * Sr:b * Sr + Sps[b]] = torch.randn(Sps[b], D, device=dev).half()
    ql = torch.tensor(Ls, dtype=torch.int32, device=dev)
    kl = torch.tensor(Sps, dtype=torch.int32, device=dev)
    out = torch.empty((B, heads), dtype=torch.float32, device=dev)
    O.pchoose_ragged(Seq(B, Lr, D, buf=q), Seq(B, Sr, D, buf=k), ql, kl, heads, 0.3, 0.2, out)
    for b in range(B):
        p = torch.empty((heads, Ls[b], Sps[b]), dtype=torch.float32, device=dev)
        _lib.check(lib.sb_pchoose(q[b * Lr:].data_ptr(), k[b * Sr:].data_ptr(), p.data_ptr(), Ls[b], Sps[b], heads, 0.3, 0.2,
                                  O._stream()), "sb_pchoose")
        assert torch.equal(out[b], p[:, -1, -1]), b
    assert torch.isfinite(out).all()


def _decide64(logits, ctl, p):
    """float64 restatement of sb_policy_decide."""
    lg, pp = logits.double().cpu().numpy(), p.double().cpu().numpy()
    res = []
    for b in range(lg.shape[0]):
        row = lg[b].copy()
        for i in ctl[b][:4]:
            if i >= 0:
                row[i] = -np.inf
        tok = int(np.argmax(row))  # first maximum
        v = np.asarray(pp[ctl[b][5]:, b, :]).reshape(-1)
        m = ctl[b][4]
        if np.isnan(v).any():
            val = np.nan  # torch's min, mean and median all give NaN
        else:
            val = v.min() if m == 0 else (math.fsum(v) / v.size if m == 1 else np.sort(v, kind="stable")[(v.size - 1) // 2])
        res.append((tok, np.float32(val)))
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("layers,heads,vocab", [(2, 2, 1126), (24, 16, 256206), (3, 5, 7)])
def test_policy_decide_matches_float64(layers, heads, vocab):
    torch.manual_seed(1)
    methods = ["min", "mean", "median"]
    B = 12
    logits = torch.randn(B, vocab + 5, device=dev)[:, :vocab]  # row stride past the vocabulary
    p = torch.rand(layers, B, heads, device=dev)
    ctl = []
    for b in range(B):
        m = methods[b % 3]
        blocked = []
        if b % 4 == 1:  # the best ids blocked: the argmax moves to the next ones
            blocked = logits[b].topk(min(4, vocab - 1)).indices.tolist()
        if b % 4 == 2:  # a tie at the maximum: the lower index wins
            j, i = sorted(torch.randperm(vocab)[:2].tolist())
            logits[b, i] = logits[b, j] = logits[b].max() + 1
        if b % 4 == 3:  # ties in the decision values, and an all-equal row
            p[:, b, :] = torch.tensor([0.25, 0.75], device=dev)[torch.arange(layers * heads, device=dev) % 2].view(layers, heads)
        if b == 7:
            p[:, b, :] = 0.5
        if b >= 9:  # a NaN decision value (min at 9, mean at 10, median at 11 and its tie row): NaN out, as torch
            p[-1, b, 0] = float("nan")
        ctl.append(O.policy_ctl(blocked, m, b % min(layers, 3), layers))
    out = O.policy_decide(logits, torch.tensor(ctl, dtype=torch.int32, device=dev), p).cpu()
    ref = _decide64(logits, ctl, p)
    for b in range(B):
        tok, bits = out[b].tolist()
        val = np.int32(bits).view(np.float32)
        assert tok == ref[b][0], (b, tok, ref[b][0])
        assert val == ref[b][1] or (np.isnan(val) and np.isnan(ref[b][1])), (b, val, ref[b][1], ctl[b])
        # and what the single-stream policy computes with torch on the same inputs
        lg = logits[b].clone()
        if ctl[b][0] >= 0:
            lg[[i for i in ctl[b][:4] if i >= 0]] = float("-inf")
        assert tok == int(lg.argmax())
        last = p[ctl[b][5]:, b, :]
        t = float({0: last.min(), 1: last.mean(), 2: last.median()}[ctl[b][4]])
        assert math.isnan(t) == bool(np.isnan(val)) and (math.isnan(t) or abs(t - float(val)) <= (1.2e-7 if ctl[b][4] == 1 else 0.0)), \
            (b, t, float(val))


@pytest.fixture(scope="module")
def tiny():
    from seamless_communication_b200.models.monotonic_decoder import load_monotonic_decoder_model
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    cfg, vc = C.tiny_v2(), C.tiny_vocoder()
    sd = S.make_unity_state_dict(cfg, 0, dec_gain=4.0, dur_gain=1.0, dur_bias=0.9)
    toks = S.make_tokenizers(cfg)
    model = load_unity_model("tiny_v2", state_dict=sd, tokenizers=toks)
    voc = load_vocoder_model("tiny", state_dict=S.make_vocoder_state_dict(vc, 1))
    mono = load_monotonic_decoder_model("tiny_v2", state_dict=S.make_monotonic_state_dict(cfg, seed=2), tokenizers=toks)
    return dict(cfg=cfg, model=model, voc=voc, mono=mono)


# (target language, duration in 320 ms segments, start tick, options)
STREAMS = [
    ("spa", 9, 0, dict(max_len_b=12)),
    ("fra", 5, 1, dict(max_len_b=12, no_early_stop=False, p_choose_start_layer=1)),
    ("deu", 12, 0, dict(max_len_b=20, decision_method="mean")),
    ("spa", 3, 4, dict(max_len_b=6, decision_method="median")),
    ("eng", 7, 2, dict(max_len_b=12, decision_threshold=0.3, no_early_stop=False, decision_method="median")),
    ("fra", 1, 3, dict(max_len_b=12)),
    ("spa", 10, 5, dict(max_len_b=4, p_choose_start_layer=-1)),  # the last layer, as p_choose[-1:]
]


@pytest.mark.gpu
def test_batched_streams_equal_each_stream_alone(tiny):
    """Streams of different durations and start ticks, with mixed target languages and options, through one
    StreamingS2STBatch: every stream's text ids (hence its READ/WRITE sequence), units and waveform chunks per tick equal
    StreamingS2ST run alone on the same audio.  Host syncs inside the policy rounds are counted by torch's sync debug mode:
    exactly one per round, the read of the decisions."""
    from seamless_communication_b200.streaming.pipeline import StreamingS2ST
    seg = 5120
    common = dict(min_starting_wait_w2vbert=40, min_unit_chunk_size=5)
    waves = [S.make_waveforms(1, n * seg - 700 * (i % 3), seed=20 + i)[0] for i, (_, n, _, _) in enumerate(STREAMS)]

    def segments(w):
        return [(w[s:s + seg], s + seg >= w.numel()) for s in range(0, w.numel(), seg)]

    alone = []
    for (lang, _, _, opt), w in zip(STREAMS, waves):
        st = StreamingS2ST(tiny["model"], tiny["mono"], tiny["voc"], lang, **common, **opt)
        alone.append([st.push(x, finished=f) for x, f in segments(w)])
    drv = StreamingS2STBatch(tiny["model"], tiny["mono"], tiny["voc"])
    ids = [drv.add_stream(lang, **common, **opt) for lang, _, _, opt in STREAMS]
    policy, per_tick = drv._policy, []

    def counted(calls):
        r0 = drv.rounds
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                policy(calls)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        syncs = [f"{w.filename}:{w.lineno}" for w in caught if "called a synchronizing CUDA operation" in str(w.message)]
        per_tick.append((drv.rounds - r0, len(syncs), syncs))

    drv._policy = counted
    segs = [segments(w) for w in waves]
    got = [[] for _ in STREAMS]
    n_ticks = max(start + len(s) for (_, _, start, _), s in zip(STREAMS, segs))
    for t in range(n_ticks):
        feed, fin = {}, set()
        for i, (_, _, start, _) in enumerate(STREAMS):
            if start <= t < start + len(segs[i]):
                x, f = segs[i][t - start]
                feed[ids[i]] = x
                if f:
                    fin.add(ids[i])
        res = drv.push(feed, finished=fin)
        for i in range(len(STREAMS)):
            if ids[i] in feed:
                got[i].append(res[ids[i]])
    assert drv.rounds == drv.host_reads and drv.rounds > 0
    assert all(syncs == rounds for rounds, syncs, _ in per_tick), [t for t in per_tick if t[0] != t[1]]
    assert sum(t[0] for t in per_tick) == drv.rounds
    wrote, max_err = 0, 0.0
    for i in range(len(STREAMS)):
        assert len(got[i]) == len(alone[i])
        for t, ((n1, u1, w1), (n2, u2, w2)) in enumerate(zip(got[i], alone[i])):
            assert n1 == n2, (i, t, n1, n2)
            assert (u1 is None) == (u2 is None) and (u1 is None or torch.equal(u1, u2)), (i, t)
            assert (w1 is None) == (w2 is None), (i, t)
            if w1 is not None:
                max_err = max(max_err, (w1.float() - w2.float()).abs().max().item())
            wrote += len(n1)
    print(f"{len(STREAMS)} streams, {n_ticks} ticks, {drv.rounds} policy rounds, {wrote} tokens; waveform max |diff| {max_err:.1e}")
    assert wrote > 0
    assert max_err == 0.0
