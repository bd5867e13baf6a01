"""N-gram repeat blocking (fairseq2's NGramRepeatBlockProcessor) in the text and AR unit searches: the processor class
and the generator's acceptance on the CPU, the oracle's restatement (tests/oracle_ngram.py) on hand-built rows,
`sb_ngram_ban_step` against that restatement, the search's integer half replayed on the oracle's logits, the engine's
searches against the oracle, and Translator.predict end to end."""
import ctypes as Ct
import math

import numpy as np
import pytest
import torch

from oracle.unity_oracle import UnityOracle
from oracle_ngram import UnityOracleNGram, ngram_bans, repeated_ngrams
from seamless_communication_b200 import config as C, synthetic as S
from seamless_communication_b200.inference import BannedSequenceProcessor, NGramRepeatBlockProcessor, SequenceGeneratorOptions
from seamless_communication_b200.models.unity.model import t2u_decoder_config, t2u_decoder_state_dict
from test_v1_s2st import _prefix, ar_state_dict, with_reachable_eos

dev = "cuda"
gpu = pytest.mark.gpu
SB_EINVAL = -1


# ------------------------------------------------------------------------------------------------ CPU: API
def test_processor_constructor_checks():
    for bad in (0, -1, -3):
        with pytest.raises(ValueError, match="greater than 0"):
            NGramRepeatBlockProcessor(bad)
    assert NGramRepeatBlockProcessor(1).ngram_size == 1
    assert NGramRepeatBlockProcessor(4).ngram_size == 4


def _generator(t2u_model, text_proc=None, unit_proc=None):
    from seamless_communication_b200.inference import UnitYGenerator
    from seamless_communication_b200.models.unity import UnitTokenizer
    cfg = C.tiny_v1()
    model = type("M", (), {"eval": lambda self: None, "text_decoder": object(), "t2u_model": t2u_model})()
    return UnitYGenerator(model, S.make_tokenizers(cfg)[0], "spa", UnitTokenizer(cfg.num_units, cfg.unit_langs, cfg.name),
                          text_opts=SequenceGeneratorOptions(step_processor=text_proc),
                          unit_opts=SequenceGeneratorOptions(step_processor=unit_proc))


def test_generator_accepts_ngram_blocking_on_text_and_ar_unit_options():
    """Text options take it on every model, AR unit options on seamlessM4T_large; any other processor still raises, and
    the NAR T2U (no search) does not read the unit options, as in the reference."""
    from seamless_communication_b200.models.unity import UnitYNART2UModel, UnitYT2UModel
    ar, nar = UnitYT2UModel.__new__(UnitYT2UModel), UnitYNART2UModel.__new__(UnitYNART2UModel)
    g = _generator(ar, NGramRepeatBlockProcessor(3), NGramRepeatBlockProcessor(2))
    assert g.text_opts.step_processor.ngram_size == 3 and g.unit_opts.step_processor.ngram_size == 2
    _generator(ar, BannedSequenceProcessor([[5]]), NGramRepeatBlockProcessor(4))
    _generator(nar, NGramRepeatBlockProcessor(3), NGramRepeatBlockProcessor(3))
    _generator(nar, None, object())
    for text_proc, unit_proc in ((object(), None), (None, object()), (None, BannedSequenceProcessor([[5]]))):
        with pytest.raises(NotImplementedError):
            _generator(ar, text_proc, unit_proc)
    with pytest.raises(NotImplementedError):
        _generator(nar, object(), None)


# ------------------------------------------------------------------------------------------------ CPU: the oracle's rule
def test_oracle_processor_on_hand_built_rows():
    """`ngram_bans(seqs[row, :step+1], n)`: prompt [3, 50] included, one entry per matching start."""
    assert ngram_bans([3, 50, 7, 8, 9, 7], 2) == [8]                  # bigram 7 8 would repeat
    assert ngram_bans([3, 50, 7, 8, 9, 7, 8], 3) == [9]               # trigram 7 8 9 would repeat
    assert ngram_bans([3, 50, 7, 8, 9, 7, 8], 2) == [9]
    assert ngram_bans([3, 50, 7, 3, 50], 3) == [7]                    # the match is the prompt itself
    assert ngram_bans([3, 50, 7, 3], 2) == [50]
    assert ngram_bans([5] * 6, 2) == [5] * 5                          # all equal: every start matches
    assert ngram_bans([5] * 6, 6) == [5]
    assert ngram_bans([1, 2, 1, 2, 1], 3) == [2]                      # periodic, overlapping occurrences
    assert ngram_bans([1, 2, 1, 2, 1], 2) == [2, 2]
    assert ngram_bans([1, 2, 3, 1, 2, 3, 1, 2], 3) == [3, 3]
    # the boundary: a row of n-1 tokens has no start; at n tokens (step n-1) the single start i = 0
    assert ngram_bans([3, 50], 3) == [] and ngram_bans([50, 50], 3) == []
    assert ngram_bans([3, 50, 50], 3) == [] and ngram_bans([50, 50, 50], 3) == [50]
    assert ngram_bans([7], 2) == [] and ngram_bans([7, 7], 2) == [7]
    # n = 1: every token the row holds, the prompt's EOS included
    assert ngram_bans([3, 50, 7, 7], 1) == [3, 50, 7, 7]
    assert ngram_bans([3], 1) == [3]
    assert repeated_ngrams([1, 2, 1, 2, 1], 2) == [(1, 2), (2, 1)] and repeated_ngrams([1, 2, 3], 2) == []


def _tiny_v2_oracle():
    cfg = C.tiny_v2()
    sd, toks = S.make_unity_state_dict(cfg, 0, dec_gain=4.0), S.make_tokenizers(cfg)
    return cfg, sd, toks, [cfg.text_eos, toks[0].lang_index("spa")]


def test_oracle_restates_the_pinned_search_and_blocks():
    """Without the processor UnityOracleNGram.beam_search is UnityOracle.beam_search step for step.  With it no hypothesis
    holds a repeated n-gram, and the random model's looping winner changes; n = 1 bans the prompt's EOS, so nothing
    finishes."""
    cfg, sd, toks, prefix = _tiny_v2_oracle()
    torch.manual_seed(5)
    enc = torch.randn(2, 12, cfg.model_dim)
    with torch.inference_mode():
        t0, t1 = {"sentence": 1}, {"sentence": 1}
        plain = UnityOracle(cfg.to_dict(), sd, toks).beam_search(enc, None, prefix, hard_max=24, trace=t0)
        on = UnityOracleNGram(cfg.to_dict(), sd, toks)
        assert on.beam_search(enc, None, prefix, hard_max=24, trace=t1) == plain
        assert [x.tolist() for x in t0["beam_idx"]] == [x.tolist() for x in t1["beam_idx"]]
        assert any(repeated_ngrams(h[1], 2) for h in plain[0])
        for n in (2, 3):
            got = on.beam_search(enc, None, prefix, hard_max=24, ngram=n)
            for b in range(2):
                assert got[b] and all(not repeated_ngrams(ids, n) for _, ids in got[b]), (n, b)
                assert got[b][0][1] != plain[b][0][1]
        assert on.beam_search(enc, None, prefix, hard_max=24, ngram=1) == [[], []]


# ------------------------------------------------------------------------------------------------ CPU: argument checks
_BASE = 1 << 24  # never dereferenced: every call below is refused before anything is launched


def test_ngram_ban_step_refuses_bad_arguments_before_any_cuda_call():
    """n < 1, a cap below the starts a row can have (seq_ld - n + 1, and at least 1), a buffer that is not 4-byte aligned
    and null pointers return SB_EINVAL, with nothing launched."""
    from seamless_communication_b200 import _lib
    lib = _lib.load()
    ok = dict(seqs=_BASE, seq_ld=40, step=_BASE + (1 << 20), rows=3, n=3, cap=38, ids=_BASE + (2 << 20), cnt=_BASE + (3 << 20))
    bad = [dict(n=0), dict(n=-2), dict(cap=37), dict(cap=0), dict(n=50, cap=0), dict(seqs=_BASE + 2), dict(ids=_BASE + 1),
           dict(cnt=_BASE + 3), dict(step=_BASE + 2), dict(seqs=0), dict(step=0), dict(rows=0), dict(seq_ld=0)]
    for kw in bad:
        a = {**ok, **kw}
        n0 = lib.sb_launch_count()
        rc = lib.sb_ngram_ban_step(a["seqs"] or None, a["seq_ld"], a["step"] or None, a["rows"], a["n"], a["cap"], a["ids"],
                                   a["cnt"], None)
        assert rc == SB_EINVAL and lib.sb_launch_count() == n0, kw
        assert b"sb_ngram_ban_step" in lib.sb_last_error()


# ------------------------------------------------------------------------------------------------ GPU: the kernel
def _stream():
    return torch.cuda.current_stream().cuda_stream


def _rows(ML, g):
    """Random and adversarial rows, each starting with the prompt [3, 50]."""
    rows = [torch.randint(4, 8, (ML,), generator=g).tolist(),        # few symbols: many matches
            torch.randint(4, 2000, (ML,), generator=g).tolist(),     # many symbols: few matches
            [9] * ML,                                                 # all equal
            [4 + t % 2 for t in range(ML)],                           # period 2
            [4 + t % 3 for t in range(ML)],                           # period 3
            ([7, 3, 50] * ML)[:ML],                                   # the prompt repeats
            ([3, 50, 11, 12] * ML)[:ML]]                              # the prompt and what follows it repeat
    for r in rows:
        r[:2] = [3, 50]
    return torch.tensor(rows, dtype=torch.int32)


@gpu
@pytest.mark.parametrize("ML", [40, 700])
def test_ngram_ban_step_matches_restatement(ML):
    """Every row's ban list equals the integer restatement (as a multiset: one id per matching start) at every step from
    0 through ML - 1 and past it (read as ML - 1), n in 1..5, step read from the device, cap at its minimum
    ML - n + 1; nothing is written past a row's count or past the last row."""
    from seamless_communication_b200 import ops
    rows = _rows(ML, torch.Generator().manual_seed(ML))
    R = rows.shape[0]
    seqs = rows.to(dev)
    steps = list(range(ML + 2)) if ML <= 64 else sorted(set(range(0, ML, 37)) | {1, 2, 3, 4, 5, ML - 2, ML - 1, ML, ML + 5})
    rl = rows.tolist()
    for n in range(1, 6):
        cap = ML - n + 1
        flat = torch.full((R * cap + 64,), -7, dtype=torch.int32, device=dev)
        ids, cnt = flat[:R * cap].view(R, cap), torch.full((R,), -1, dtype=torch.int32, device=dev)
        step = torch.zeros(1, dtype=torch.int32, device=dev)
        for t in steps:
            flat.fill_(-7)
            step.fill_(t)
            ops.ngram_ban_step(seqs, step, n, ids, cnt)
            got_n, got = cnt.tolist(), ids.cpu()
            tail = flat[R * cap:]
            assert bool((tail == -7).all()), (n, t)
            te = min(t, ML - 1)
            for r in range(R):
                want = ngram_bans(rl[r][:te + 1], n)
                assert got_n[r] == len(want), (n, t, r)
                assert sorted(got[r, :got_n[r]].tolist()) == sorted(want), (n, t, r)
                assert bool((got[r, got_n[r]:] == -7).all()), (n, t, r)


# ------------------------------------------------------------------------------------------------ GPU: search replay
def _replay_with_ngram(cfg, trace, prefix, beam, V, n, tiles=False, unk_penalty=0.0):
    """The integer half of a blocking step (sb_ngram_ban_step -> ban-aware top-K -> sb_beam_step -> sb_step_advance, as
    engine._decoder_step_select with `ngram`) on the oracle's fp32 logits, one sentence.  Returns (parents, tokens) per
    step and the finished hypotheses in finalisation order."""
    from seamless_communication_b200 import _lib
    from seamless_communication_b200._lib import BeamDesc, check
    from test_mintox import _tile_stats
    lib, st = _lib.load(), _stream()
    ML, P, R, c = trace["max_len"], len(prefix), beam, cfg
    K = min(2 * beam + 1, 16)
    ld = (V + 7) // 8 * 8
    i32 = dict(dtype=torch.int32, device=dev)
    seqs, anc = torch.zeros((R, ML), **i32), torch.arange(R, **i32)[:, None].repeat(1, ML).contiguous()
    seqs[:, :P] = torch.tensor(prefix, **i32)
    scores = torch.zeros((R, ML), device=dev)
    scores[:, :P] = trace["prefix_scores"].to(dev)
    step = torch.full((1,), P - 1, **i32)
    logits = torch.zeros((R, ld), device=dev)
    cv, ci, el = torch.empty((R, K), device=dev), torch.empty((R, K), **i32), torch.empty((R,), device=dev)
    cap = ML
    bids, bn = torch.zeros((R, cap), **i32), torch.zeros((R,), **i32)
    fin = dict(count=torch.zeros(1, **i32), score=torch.full((1, beam), -math.inf, device=dev), len=torch.zeros((1, beam), **i32),
               seqs=torch.zeros((1, beam, ML), **i32), active=torch.ones(1, **i32), n_active=torch.ones(1, **i32),
               anc=torch.zeros((1, beam, ML), **i32))
    d = BeamDesc()
    d.batch, d.beam, d.max_len, d.vocab, d.K = 1, beam, ML, V, K
    d.step_ptr, d.prefix_len, d.eos_idx, d.min_len, d.len_penalty = step.data_ptr(), P, c.text_eos, 1, 1.0
    d.cand_val, d.cand_idx, d.eos_lprob = cv.data_ptr(), ci.data_ptr(), el.data_ptr()
    d.seqs, d.scores, d.anc = seqs.data_ptr(), scores.data_ptr(), anc.data_ptr()
    d.fin_count, d.fin_score, d.fin_len = fin["count"].data_ptr(), fin["score"].data_ptr(), fin["len"].data_ptr()
    d.fin_seqs, d.active, d.n_active, d.fin_anc = fin["seqs"].data_ptr(), fin["active"].data_ptr(), fin["n_active"].data_ptr(), fin["anc"].data_ptr()
    decisions = []
    for s, lg in enumerate(trace["logits"]):
        pos = P - 1 + s
        assert seqs[:, pos].tolist() == trace["inputs"][s].tolist(), f"step {s}: device rows feed other tokens than the oracle's"
        logits[:, :V] = lg.to(dev)
        check(lib.sb_ngram_ban_step(seqs.data_ptr(), ML, step.data_ptr(), R, n, cap, bids.data_ptr(), bn.data_ptr(), st))
        if tiles:
            stats = _tile_stats(logits, V)
            check(lib.sb_logits_topk_tiles_ban(logits.data_ptr(), ld, stats.data_ptr(), R, V, c.text_pad, c.text_eos, c.text_unk,
                                               unk_penalty, K, cv.data_ptr(), ci.data_ptr(), el.data_ptr(), bids.data_ptr(),
                                               bn.data_ptr(), cap, st))
        else:
            check(lib.sb_logits_topk_ban(logits.data_ptr(), ld, R, V, c.text_pad, c.text_eos, c.text_unk, unk_penalty, K,
                                         cv.data_ptr(), ci.data_ptr(), el.data_ptr(), bids.data_ptr(), bn.data_ptr(), cap, st))
        check(lib.sb_beam_step(Ct.byref(d), st))
        check(lib.sb_step_advance(step.data_ptr(), st))
        if int(fin["active"].item()) == 0:
            break
        decisions.append((anc[:, pos].tolist(), seqs[:, pos + 1].tolist()))
    n_fin = int(fin["count"].item())
    return decisions, [(float(fin["score"][0, j]), fin["seqs"][0, j, :int(fin["len"][0, j])].tolist()) for j in range(n_fin)]


_TRACES = {}


def _blocked_trace(kind, beam, n, eos_scale):
    """The oracle's blocking search (and its plain search) on one sentence: tiny_v2 text (1 126 tokens) or the tiny_v1
    AR unit decoder (338 units).  `eos_scale` 0: the synthetic weights score EOS 0, so every hypothesis runs to the
    forced EOS at the budget; otherwise an EOS row that ends hypotheses early (test_v1_s2st.with_reachable_eos)."""
    key = (kind, beam, n, eos_scale)
    if key not in _TRACES:
        if kind == "text":
            cfg, sd, toks, prefix = _tiny_v2_oracle()
            sd = with_reachable_eos(sd, cfg, eos_scale, text=True) if eos_scale else sd
            oracle, dcfg, soft, hard, unk = UnityOracleNGram(cfg.to_dict(), sd, toks), cfg, (1, 200), 30, -11.0
        else:
            cfg = C.tiny_v1()
            sd = with_reachable_eos(ar_state_dict(), cfg, eos_scale) if eos_scale else ar_state_dict()
            dcfg = t2u_decoder_config(cfg)
            oracle, prefix, soft, hard, unk = UnityOracleNGram(dcfg.to_dict(), t2u_decoder_state_dict(sd)), _prefix(cfg), (25, 50), 40, 0.0
        torch.manual_seed(17 + beam)
        enc = torch.randn(1, 11, cfg.model_dim)
        trace = {"sentence": 0}
        with torch.inference_mode():
            plain = oracle.beam_search(enc, None, prefix, beam=beam, soft_max=soft, hard_max=hard, unk_penalty=unk)
            oracle.beam_search(enc, None, prefix, beam=beam, soft_max=soft, hard_max=hard, unk_penalty=unk, trace=trace, ngram=n)
        _TRACES[key] = (dcfg, prefix, trace, plain[0], unk)
    return _TRACES[key]


@gpu
@pytest.mark.parametrize("eos_scale", [0.0, 1.5])
@pytest.mark.parametrize("tiles", [False, True])
@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("beam", [2, 5])
@pytest.mark.parametrize("kind", ["text", "units"])
def test_blocking_search_replay_is_bit_exact_on_oracle_logits(kind, beam, n, tiles, eos_scale):
    """sb_ngram_ban_step -> `_ban` top-K -> sb_beam_step on UnityOracleNGram.beam_search's own fp32 logits: parents, tokens
    and the finished hypotheses equal the oracle's at every step, and no finished hypothesis holds a repeated n-gram.
    Searches that run to the budget loop on the random weights, so there the blocking must have changed the outcome."""
    cfg, prefix, trace, plain, unk = _blocked_trace(kind, beam, n, eos_scale)
    decisions, finished = _replay_with_ngram(cfg, trace, prefix, beam, cfg.text_vocab, n, tiles=tiles, unk_penalty=unk)
    assert len(decisions) == len(trace["beam_idx"])
    for s, (parents, toks) in enumerate(decisions):
        assert parents == trace["beam_idx"][s].tolist(), f"step {s}: parent beams differ"
        if s + 1 < len(trace["inputs"]):
            assert toks == trace["inputs"][s + 1].tolist(), f"step {s}: tokens differ"
    assert [f[1] for f in finished] == [f[1] for f in trace["finished"]]
    assert np.allclose([f[0] for f in finished], [f[0] for f in trace["finished"]], rtol=0, atol=1e-5)
    assert finished and all(not repeated_ngrams(ids, n) for _, ids in finished)
    if not eos_scale:
        assert sorted(f[1] for f in finished) != sorted(h[1] for h in plain)


# ------------------------------------------------------------------------------------------------ GPU: engine searches
@pytest.fixture(scope="module")
def tiny_v2():
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    cfg, sd, toks, prefix = _tiny_v2_oracle()
    return dict(cfg=cfg, toks=toks, prefix=prefix, model=load_unity_model("tiny_v2", state_dict=sd, tokenizers=toks),
                voc=load_vocoder_model("tiny", state_dict=S.make_vocoder_state_dict(C.tiny_vocoder(), 1)),
                uo=UnityOracleNGram(cfg.to_dict(), sd, toks))


@pytest.fixture(scope="module")
def tiny_v1():
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    cfg = C.tiny_v1()
    sd = with_reachable_eos(ar_state_dict(), cfg, 1.5)
    toks = S.make_tokenizers(cfg)
    dcfg = t2u_decoder_config(cfg)
    return dict(cfg=cfg, model=load_unity_model("tiny_v1", state_dict=sd, tokenizers=toks),
                voc=load_vocoder_model("tiny", state_dict=S.make_vocoder_state_dict(C.tiny_vocoder(), seed=1, dur_predictor=True)),
                ou=UnityOracleNGram(dcfg.to_dict(), t2u_decoder_state_dict(sd)))


def _audit(o, enc_b, hyp, ref_best):
    """Same hypothesis, or a near tie under the oracle's own scoring (oracle/ASSUMPTIONS.md #9)."""
    if hyp[1] == ref_best[1]:
        return
    ids = torch.tensor(hyp[1])[None]
    lp = torch.log_softmax(o.project(o.decoder(o.embed_text(ids[:, :-1], 0), enc_b, None)).float(), -1)[0]
    sc = sum(float(lp[t, ids[0, t + 1]]) for t in range(ids.shape[1] - 1)) / (ids.shape[1] - 1)
    assert abs(sc - ref_best[0]) < 2e-2, (sc, ref_best[0])


@gpu
def test_engine_text_search_blocks_and_matches_oracle(tiny_v2):
    """engine.beam_search(ngram=n) through its captured graph equals the oracle's blocking search on the same encoder
    output (or is a near tie under the oracle's scoring: the engine's logits are fp16 products, see
    test_blocking_search_replay_is_bit_exact_on_oracle_logits for the exact comparison), holds no repeated n-gram in any
    hypothesis, launches one kernel more per step than the plain select graph, and leaves the plain search's graphs and
    results alone."""
    from seamless_communication_b200.ops import Seq
    cfg, uo, eng, prefix = tiny_v2["cfg"], tiny_v2["uo"], tiny_v2["model"].engine, tiny_v2["prefix"]
    torch.manual_seed(9)
    enc = torch.randn(3, 16, cfg.model_dim).half().float()
    e = Seq(3, 16, cfg.model_dim, buf=enc.to(dev).half().reshape(-1, cfg.model_dim).contiguous())
    plain = eng.beam_search(e, None, prefix, beam=5, hard_max=24)
    st = eng._last_search_state
    g_fwd, g_sel, k0 = st["g_fwd"], st["g_sel"], eng.graph_kernels
    eng.beam_search(e, None, prefix, beam=5, hard_max=24)
    k_plain = eng.graph_kernels - k0
    for n in (2, 3, 4):
        got = eng.beam_search(e, None, prefix, beam=5, hard_max=24, ngram=n)
        assert eng._last_search_state is st and st["n_sel_ngram"] == st["n_sel"] + 1
        with torch.inference_mode():
            ref = uo.beam_search(enc, None, prefix, beam=5, hard_max=24, ngram=n)
        for b in range(3):
            assert got[b] and all(not repeated_ngrams(ids, n) for _, ids in got[b]), (n, b)
            if repeated_ngrams(plain[b][0][1], n):
                assert got[b][0][1] != plain[b][0][1]
            with torch.inference_mode():
                _audit(uo, enc[b:b + 1], got[b][0], ref[b][0])
    k1 = eng.graph_kernels
    assert eng.beam_search(e, None, prefix, beam=5, hard_max=24) == plain
    assert eng.graph_kernels - k1 == k_plain
    assert st["g_fwd"] is g_fwd and st["g_sel"] is g_sel  # blocking never recaptures the plain graphs
    with pytest.raises(ValueError):
        eng.beam_search(e, None, prefix, beam=5, hard_max=24, ngram=0)
    with pytest.raises(NotImplementedError):
        eng.beam_search(e, None, prefix, beam=5, hard_max=24, ngram=2, banned=[[5]])


@gpu
def test_engine_unit_search_blocks_and_matches_oracle(tiny_v1):
    """The AR unit search of tiny_v1 with blocking: the oracle's hypotheses (or near ties), no repeated n-gram, and the
    plain unit search unchanged afterwards."""
    from seamless_communication_b200.ops import Seq
    cfg, ou, t2u = tiny_v1["cfg"], tiny_v1["ou"], tiny_v1["model"].t2u_model
    lens = [11, 6]
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 11, cfg.model_dim, generator=g).half()
    x[1, 6:] = 0
    e = Seq(2, 11, cfg.model_dim, buf=x.to(dev).view(22, -1))
    el = torch.tensor(lens, dtype=torch.int32, device=dev)
    prefix = _prefix(cfg)
    plain = t2u.beam_search(e, el, prefix, beam=5, soft_max=(25, 50), hard_max=48)
    for n in (2, 3):
        got = t2u.beam_search(e, el, prefix, beam=5, soft_max=(25, 50), hard_max=48, ngram=n)
        with torch.inference_mode():
            ref = ou.beam_search(x.float(), torch.tensor(lens), prefix, beam=5, soft_max=(25, 50), hard_max=48, ngram=n)
        for b in range(2):
            assert got[b] and all(not repeated_ngrams(ids, n) for _, ids in got[b]), (n, b)
            if repeated_ngrams(plain[b][0][1], n):
                assert got[b][0][1] != plain[b][0][1]
            with torch.inference_mode():
                _audit(ou, x[b:b + 1, :lens[b]].float(), got[b][0], ref[b][0])
    assert t2u.beam_search(e, el, prefix, beam=5, soft_max=(25, 50), hard_max=48) == plain


# ------------------------------------------------------------------------------------------------ GPU: end to end
def _hyps():
    from seamless_communication_b200.inference import Translator
    return Translator._tls.generator


@gpu
@pytest.mark.parametrize("task", ["s2tt", "s2st"])
def test_translator_predict_with_ngram_blocking_tiny_v2(tiny_v2, task):
    """Translator.predict with text_generation_opts=SequenceGeneratorOptions(step_processor=NGramRepeatBlockProcessor(3)):
    the text hypotheses hold no repeated trigram, and differ from the plain ones exactly when those repeat one; a later
    plain predict returns the plain outputs bit for bit."""
    from seamless_communication_b200.inference import Translator
    tr = Translator(tiny_v2["model"], tiny_v2["voc"], device="cuda:0")
    src = tr.fbank_batch(S.make_waveforms(3, 32000, seed=21))
    plain_opts = SequenceGeneratorOptions(hard_max_seq_len=20)
    opts = SequenceGeneratorOptions(hard_max_seq_len=20, step_processor=NGramRepeatBlockProcessor(3))
    texts0, speech0 = tr.predict(src, task, "spa", text_generation_opts=plain_opts)
    plain_hyps = [h[0][1] for h in _hyps().last_text_output.hypotheses]
    texts, speech = tr.predict(src, task, "spa", text_generation_opts=opts)
    hyps = [h[0][1] for h in _hyps().last_text_output.hypotheses]
    assert opts.step_processor.ngram_size == 3 and len(texts) == 3
    assert all(not repeated_ngrams(h, 3) for h in hyps)
    assert any(repeated_ngrams(h, 3) for h in plain_hyps) == (hyps != plain_hyps)
    if task == "s2st":
        assert len(speech.units) == 3 and all(len(u) > 0 for u in speech.units)
    texts1, speech1 = tr.predict(src, task, "spa", text_generation_opts=plain_opts)
    assert texts1 == texts0
    if task == "s2st":
        assert speech1.units == speech0.units
        assert all(torch.equal(a, b) for a, b in zip(speech1.audio_wavs, speech0.audio_wavs))


@gpu
def test_translator_predict_with_text_and_unit_blocking_tiny_v1(tiny_v1):
    """seamlessM4T_large-type S2ST with blocking on both searches: no repeated trigram in the text hypotheses, none of
    size 4 in the unit hypotheses, and the unit search changed exactly when the plain one repeated a 4-gram."""
    from seamless_communication_b200.inference import Translator
    tr = Translator(tiny_v1["model"], tiny_v1["voc"], device="cuda:0")
    src = tr.fbank_batch(S.make_waveforms(2, 32000, seed=4))
    opts = SequenceGeneratorOptions(hard_max_seq_len=20, step_processor=NGramRepeatBlockProcessor(3))
    uplain = SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40)
    uopts = SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40, step_processor=NGramRepeatBlockProcessor(4))
    tr.predict(src, "s2st", "spa", text_generation_opts=opts, unit_generation_opts=uplain)
    plain_units = [h[0][1] for h in _hyps().last_unit_output["hypotheses"]]
    texts, speech = tr.predict(src, "s2st", "spa", text_generation_opts=opts, unit_generation_opts=uopts)
    gen = _hyps()
    assert all(not repeated_ngrams(h[0][1], 3) for h in gen.last_text_output.hypotheses)
    units = [h[0][1] for h in gen.last_unit_output["hypotheses"]]
    assert all(not repeated_ngrams(u, 4) for u in units)
    assert any(repeated_ngrams(u, 4) for u in plain_units) == (units != plain_units)
    assert len(speech.audio_wavs) == 2 and all(w.numel() > 0 for w in speech.audio_wavs)
