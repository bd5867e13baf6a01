"""MinTox: the ETOX added-toxicity check against the reference's own code (tests/golden/mintox_etox.json, made by
make_golden_mintox.py), the banned-sequence kernels against Python / float64 restatements, the search with bans against
the oracle, and the re-decode through Translator.predict."""
import ctypes as Ct
import json
import math
import os
import sys

import pytest
import torch

from seamless_communication_b200 import config as C, synthetic as S
from seamless_communication_b200.inference import BannedSequenceProcessor, SequenceGeneratorOptions

G = os.path.join(os.path.dirname(__file__), "golden")
sys.path.insert(0, G)
from make_golden_mintox import StubSpEncoder  # noqa: E402

FIX = json.load(open(os.path.join(G, "mintox_etox.json"), encoding="utf-8"))
dev = "cuda"
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ CPU: ETOX and helpers
@pytest.fixture()
def checker(tmp_path):
    from seamless_communication_b200.toxicity import load_etox_bad_word_checker
    for name, text in FIX["files"].items():
        (tmp_path / name).write_text(text, encoding="utf-8")
    return load_etox_bad_word_checker("mintox", dataset_dir=str(tmp_path), sp_encoder=StubSpEncoder())


def test_card_tables_match_the_mintox_card():
    assert list(C.MINTOX_ETOX_LANG_VARIANTS) == FIX["etox_lang_variants"]
    assert list(C.MINTOX_SP_LANGS) == FIX["sp_langs"]


def test_loader_reproduces_the_reference_word_lists(checker):
    assert {k: sorted(v) for k, v in checker.bad_words.items()} == FIX["bad_words"]
    assert checker.bad_word_variants == FIX["bad_word_variants"]
    assert checker.sp_langs == set(FIX["sp_langs"])


def test_get_and_extract_bad_words_match_the_reference(checker):
    for text, lang, want in FIX["get_bad_words"]:
        assert sorted(checker.get_bad_words(text, lang)) == want, (text, lang)
    for src, tgt, sl, tl, want, err in FIX["extract_bad_words"]:
        if err is None:
            assert sorted(checker.extract_bad_words(src, tgt, sl, tl)) == want, (src, tgt)
        else:
            with pytest.raises(KeyError):
                checker.extract_bad_words(src, tgt, sl, tl)
    with pytest.raises(RuntimeError) as e:
        checker.get_bad_words("abcd", "xyz")
    assert str(e.value) == FIX["unsupported_error"]


def test_loader_refuses_to_download():
    from seamless_communication_b200.toxicity import load_etox_bad_word_checker
    with pytest.raises(ValueError, match="dataset_dir"):
        load_etox_bad_word_checker("mintox")
    with pytest.raises(ValueError):
        load_etox_bad_word_checker("mutox", dataset_dir=".")


def test_mintox_helpers_match_the_reference(checker):
    from seamless_communication_b200.models.unity import UnitTokenizer
    from seamless_communication_b200.toxicity import mintox as M
    b = FIX["batch_indices"]
    words, idx = M._extract_bad_words_with_batch_indices(b["src"], b["tgt"], "eng", "spa", checker)
    assert sorted(words) == b["words"] and idx == b["indices"]
    r = FIX["replace_text"]
    texts = ["t0", "t1", "t2", "t3", "t4"]
    M._replace_with_new_text_output_in_batch(texts, r["indices"], r["new"])
    assert texts == r["result"]
    ut = UnitTokenizer(100, ["eng"], "nar_multilingual_v2")
    for case in FIX["replace_units"]:
        orig, new = torch.tensor(case["original"]), torch.tensor(case["new"])
        got = M._replace_with_new_unit_output_in_batch(ut, orig, torch.tensor(case["indices"]), new)
        if new.size(1) <= orig.size(1):  # the reference merges in place
            assert got.tolist() == case["original_after"]
        else:  # the reference pads a local copy and drops it (its batch keeps the old units); here the merge is returned
            assert case["original_after"] == case["original"]
            want = torch.nn.functional.pad(torch.tensor(case["original"]), (0, new.size(1) - orig.size(1)), value=1)
            want[case["indices"]] = new
            assert got.tolist() == want.tolist()


def test_banned_sequence_processor_and_raw_encoder():
    with pytest.raises(ValueError):
        BannedSequenceProcessor([])
    with pytest.raises(ValueError):
        BannedSequenceProcessor([[3], []])
    p = BannedSequenceProcessor([torch.tensor([5, 6]), [7]])
    assert p.banned_seqs == [[5, 6], [7]]
    tok = S.make_tokenizers(C.tiny_v2())[0]
    enc = tok.create_raw_encoder()
    w = tok.model.index_to_token(40)[1:]
    assert enc(w).tolist() == [40]
    assert enc("★" + w).tolist() == [tok.vocab_info.unk_idx, 40]
    assert enc("zzzzzz").tolist() == [tok.vocab_info.unk_idx]
    from seamless_communication_b200.toxicity.mintox import banned_sequence_processor
    assert banned_sequence_processor(tok, [w, w]).banned_seqs == [[40], [40]]


def test_generator_accepts_only_the_banned_sequence_processor():
    from seamless_communication_b200.inference import UnitYGenerator
    model = type("M", (), {"eval": lambda self: None, "text_decoder": object(), "t2u_model": None})()
    with pytest.raises(NotImplementedError):
        UnitYGenerator(model, None, "spa", text_opts=SequenceGeneratorOptions(step_processor=object()))


def test_translator_mintox_needs_a_checker():
    from seamless_communication_b200.inference import Translator
    with pytest.raises(ValueError, match="load_etox_bad_word_checker"):
        Translator("seamlessM4T_v2_tiny", None, device="cuda:0", apply_mintox=True)


def test_banned_oracle_restates_the_pinned_search():
    """Without bans, UnityOracleBanned.beam_search is UnityOracle.beam_search step for step; with a ban on the winner's
    first token, no hypothesis takes it."""
    from oracle.unity_oracle import UnityOracle
    from oracle_mintox import UnityOracleBanned
    cfg = C.tiny_v2()
    sd, toks = S.make_unity_state_dict(cfg, 0, dec_gain=4.0), S.make_tokenizers(cfg)
    prefix = [cfg.text_eos, toks[0].lang_index("spa")]
    torch.manual_seed(5)
    enc = torch.randn(2, 12, cfg.model_dim)
    with torch.inference_mode():
        for min_len in (1, 22):
            t0, t1 = {"sentence": 1}, {"sentence": 1}
            a = UnityOracle(cfg.to_dict(), sd, toks).beam_search(enc, None, prefix, hard_max=24, min_seq_len=min_len, trace=t0)
            ob = UnityOracleBanned(cfg.to_dict(), sd, toks)
            assert ob.beam_search(enc, None, prefix, hard_max=24, min_seq_len=min_len, trace=t1) == a
            assert [x.tolist() for x in t0["beam_idx"]] == [x.tolist() for x in t1["beam_idx"]]
            w = a[0][0][1][2]
            got = ob.beam_search(enc, None, prefix, hard_max=24, min_seq_len=min_len, banned=[[w]])
            assert got[0] and all(h[1][2] != w for h in got[0])


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _lib():
    from seamless_communication_b200 import _lib as L
    return L.load(), L.check


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _table(seqs, cap, width):
    t = torch.zeros(1 + cap + cap * width, dtype=torch.int32)
    t[0] = len(seqs)
    for j, s in enumerate(seqs):
        t[1 + j] = len(s)
        t[1 + cap + j * width + width - len(s):1 + cap + (j + 1) * width] = torch.tensor(s, dtype=torch.int32)
    return t.to(dev)


def _bans_py(row, step, seqs):
    hist = row[:step + 1]
    return sorted(s[-1] for s in seqs if len(s) == 1 or (len(s) - 1 <= len(hist) and hist[len(hist) - len(s) + 1:] == s[:-1]))


def _ban_step(seqs_t, step, table, cap, width):
    lib, check = _lib()
    R, ML = seqs_t.shape
    ids = torch.full((R, cap), -7, dtype=torch.int32, device=dev)
    n = torch.full((R,), -1, dtype=torch.int32, device=dev)
    st = torch.tensor([step], dtype=torch.int32, device=dev)
    check(lib.sb_ban_step(seqs_t.data_ptr(), ML, st.data_ptr(), R, table.data_ptr(), cap, width, ids.data_ptr(), n.data_ptr(),
                          _stream()), "sb_ban_step")
    torch.cuda.synchronize()
    return [sorted(ids[r, :int(n[r])].tolist()) for r in range(R)]


@gpu
def test_ban_step_matches_python():
    g = torch.Generator().manual_seed(3)
    R, ML = 6, 24
    rows = torch.randint(4, 9, (R, ML), generator=g, dtype=torch.int32)
    rows[:, 0], rows[:, 1] = 3, 50  # the prompt [eos, lang]
    rl = rows.tolist()
    seqs = [[5], [5], [8, 6], [3, 50, 7], [50, rl[0][2]], [rl[1][3], rl[1][4], 9], [rl[2][1], rl[2][2], rl[2][3], rl[2][4], 11],
            [4] * 30, [6, 6], [7, 7, 7]]
    width = 32
    for step in (0, 1, 2, 4, 9, 22):
        table = _table(seqs, 16, width)
        got = _ban_step(rows.to(dev), step, table, 16, width)
        assert got == [_bans_py(rl[r], step, seqs) for r in range(R)], f"step {step}"
    assert _ban_step(rows.to(dev), 5, _table([], 16, 4), 16, 4) == [[]] * R
    big = [[int(x) for x in torch.randint(4, 9, (1 + j % 3,), generator=g)] for j in range(4096)]
    got = _ban_step(rows.to(dev), 7, _table(big, 4096, 4), 4096, 4)
    assert got == [_bans_py(rl[r], 7, big) for r in range(R)]
    assert max(len(x) for x in got) > 500


def _tile_stats(lg, V):
    R = lg.shape[0]
    nt = (V + 127) // 128
    x = torch.full((R, nt * 128), -math.inf, device=dev)
    x[:, :V] = lg[:, :V]
    x = x.view(R, nt, 128)
    m = x.max(-1).values
    s = torch.exp(x - m[..., None]).sum(-1)
    return torch.stack([m, s], -1).transpose(0, 1).contiguous()  # [tile][row][2]


def _topk(lg, V, K, pad, eos, unk, pen, bans=None, tiles=False, stats=None):
    """`stats`: the tile statistics of `lg` for the tile path (default: _tile_stats)."""
    lib, check = _lib()
    R, ld = lg.shape
    cv = torch.empty((R, K), device=dev)
    ci = torch.empty((R, K), dtype=torch.int32, device=dev)
    el = torch.empty((R,), device=dev)
    if tiles and stats is None:
        stats = _tile_stats(lg, V)
    if bans is None:
        if tiles:
            check(lib.sb_logits_topk_tiles(lg.data_ptr(), ld, stats.data_ptr(), R, V, pad, eos, unk, pen, K, cv.data_ptr(), ci.data_ptr(),
                                           el.data_ptr(), _stream()))
        else:
            check(lib.sb_logits_topk(lg.data_ptr(), ld, R, V, pad, eos, unk, pen, K, cv.data_ptr(), ci.data_ptr(), el.data_ptr(), _stream()))
    else:
        cap = max(1, max(len(b) for b in bans))
        ids = torch.zeros((R, cap), dtype=torch.int32)
        for r, b in enumerate(bans):
            ids[r, :len(b)] = torch.tensor(b, dtype=torch.int32)
        ids = ids.to(dev)
        n = torch.tensor([len(b) for b in bans], dtype=torch.int32, device=dev)
        if tiles:
            check(lib.sb_logits_topk_tiles_ban(lg.data_ptr(), ld, stats.data_ptr(), R, V, pad, eos, unk, pen, K, cv.data_ptr(),
                                               ci.data_ptr(), el.data_ptr(), ids.data_ptr(), n.data_ptr(), cap, _stream()))
        else:
            check(lib.sb_logits_topk_ban(lg.data_ptr(), ld, R, V, pad, eos, unk, pen, K, cv.data_ptr(), ci.data_ptr(), el.data_ptr(),
                                         ids.data_ptr(), n.data_ptr(), cap, _stream()))
    torch.cuda.synchronize()
    return cv.cpu(), ci.cpu(), el.cpu()


@gpu
@pytest.mark.parametrize("tiles", [False, True])
@pytest.mark.parametrize("V", [1126, 256102])
def test_topk_ban_matches_float64(tiles, V):
    """Candidates in (lprob desc, id asc) order among the ids that are neither PAD nor banned, lprobs against a float64
    log-sum-exp over the WHOLE row; eos_lprob -inf when EOS is banned; an empty list equals the unbanned entry bit for bit."""
    pad, eos, unk, pen, K = 0, 3, 1, 0.5, 11
    R, ld = 6, (V + 7) // 8 * 8
    g = torch.Generator().manual_seed(V)
    lg = torch.zeros((R, ld))
    lg[:, :V] = torch.randn(R, V, generator=g) * 3
    lg = lg.to(dev)
    x = lg[:, :V].cpu()
    nt = (V + 127) // 128
    tmax = x[:, :nt * 128 - 128].reshape(R, nt - 1, 128).argmax(-1) + torch.arange(nt - 1) * 128  # argmax of full tiles
    order = x.argsort(-1, descending=True)
    bans = [
        [],                                                              # empty
        [int(order[1, 0]), int(tmax[1, 5]), int(tmax[1, 7])],            # banned tile maxima, the row's best among them
        [int(t) for t in tmax[2][x[2, tmax[2]].argsort(descending=True)[:K + 2]]],  # every one of the top K+2 tile maxima
        [eos, int(order[3, 2])],                                         # EOS banned
        [int(t) for t in order[4, :600]] + [int(t) for t in order[4, :50]],  # > 500 bans (duplicates included)
        [int(t) for t in order[5, :3]] + [pad, unk],
    ]
    cv, ci, el = _topk(lg, V, K, pad, eos, unk, pen, bans=bans, tiles=tiles)
    cv0, ci0, el0 = _topk(lg, V, K, pad, eos, unk, pen, tiles=tiles)
    assert torch.equal(cv[0], cv0[0]) and torch.equal(ci[0], ci0[0]) and torch.equal(el[0], el0[0])
    xd = x.double()
    lse = torch.logsumexp(xd, -1)
    for r in range(R):
        cand = x[r].clone()
        cand[unk] = cand[unk] - pen  # fp32, as the kernel
        cand[pad] = -math.inf
        cand[bans[r]] = -math.inf
        vals = cand.double()
        ids = sorted(range(V), key=lambda i: (-vals[i].item(), i))[:K] if V < 5000 else \
            sorted(torch.topk(vals, K + 8).indices.tolist(), key=lambda i: (-vals[i].item(), i))[:K]
        assert ci[r].tolist() == ids, f"row {r}"
        assert torch.allclose(cv[r].double(), vals[ids] - lse[r], atol=2e-5, rtol=0), f"row {r}"
        if eos in bans[r]:
            assert el[r].item() == -math.inf
        else:
            assert abs(el[r].item() - (xd[r, eos] - lse[r]).item()) < 2e-5
            assert el[r].item() == el0[r].item()
        assert not set(ci[r].tolist()) & set(bans[r])


# ------------------------------------------------------------------------------------------------ GPU: search vs oracle
def _replay_with_bans(eng, trace, prefix, beam, V, banned, min_len, tiles):
    """The integer half of the search (sb_ban_step -> ban-aware top-K -> sb_beam_step -> sb_step_advance, as
    engine._decoder_step_select with bans) on the oracle's fp32 logits, one sentence."""
    from seamless_communication_b200._lib import BeamDesc
    lib, check = _lib()
    st = _stream()
    ML, P, R, c = trace["max_len"], len(prefix), beam, eng.cfg
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
    cap, width = 16, 8
    table = _table(banned, cap, width)
    bids, bn = torch.zeros((R, cap), **i32), torch.zeros((R,), **i32)
    fin = dict(count=torch.zeros(1, **i32), score=torch.full((1, beam), -math.inf, device=dev), len=torch.zeros((1, beam), **i32),
               seqs=torch.zeros((1, beam, ML), **i32), active=torch.ones(1, **i32), n_active=torch.ones(1, **i32),
               anc=torch.zeros((1, beam, ML), **i32))
    d = BeamDesc()
    d.batch, d.beam, d.max_len, d.vocab, d.K = 1, beam, ML, V, K
    d.step_ptr, d.prefix_len, d.eos_idx, d.min_len, d.len_penalty = step.data_ptr(), P, c.text_eos, min_len, 1.0
    d.cand_val, d.cand_idx, d.eos_lprob = cv.data_ptr(), ci.data_ptr(), el.data_ptr()
    d.seqs, d.scores, d.anc = seqs.data_ptr(), scores.data_ptr(), anc.data_ptr()
    d.fin_count, d.fin_score, d.fin_len = fin["count"].data_ptr(), fin["score"].data_ptr(), fin["len"].data_ptr()
    d.fin_seqs, d.active, d.n_active, d.fin_anc = fin["seqs"].data_ptr(), fin["active"].data_ptr(), fin["n_active"].data_ptr(), fin["anc"].data_ptr()
    decisions = []
    for s, lg in enumerate(trace["logits"]):
        pos = P - 1 + s
        logits[:, :V] = lg.to(dev)
        check(lib.sb_ban_step(seqs.data_ptr(), ML, step.data_ptr(), R, table.data_ptr(), cap, width, bids.data_ptr(), bn.data_ptr(), st))
        if tiles:
            stats = _tile_stats(logits, V)
            check(lib.sb_logits_topk_tiles_ban(logits.data_ptr(), ld, stats.data_ptr(), R, V, c.text_pad, c.text_eos, c.text_unk, 0.0, K,
                                               cv.data_ptr(), ci.data_ptr(), el.data_ptr(), bids.data_ptr(), bn.data_ptr(), cap, st))
        else:
            check(lib.sb_logits_topk_ban(logits.data_ptr(), ld, R, V, c.text_pad, c.text_eos, c.text_unk, 0.0, K, cv.data_ptr(),
                                         ci.data_ptr(), el.data_ptr(), bids.data_ptr(), bn.data_ptr(), cap, st))
        check(lib.sb_beam_step(Ct.byref(d), st))
        check(lib.sb_step_advance(step.data_ptr(), st))
        if int(fin["active"].item()) == 0:
            break
        decisions.append((anc[:, pos].tolist(), seqs[:, pos + 1].tolist(), scores[:, pos + 1].tolist()))
    n = int(fin["count"].item())
    return decisions, [(float(fin["score"][0, j]), fin["seqs"][0, j, :int(fin["len"][0, j])].tolist()) for j in range(n)]


@pytest.fixture(scope="module")
def tiny_v2():
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    from oracle_mintox import UnityOracleBanned
    cfg, vc = C.tiny_v2(), C.tiny_vocoder()
    sd = S.make_unity_state_dict(cfg, 0, dec_gain=4.0, dur_gain=1.0, dur_bias=0.9)
    toks = S.make_tokenizers(cfg)
    return dict(cfg=cfg, toks=toks, model=load_unity_model("tiny_v2", state_dict=sd, tokenizers=toks),
                voc=load_vocoder_model("tiny", state_dict=S.make_vocoder_state_dict(vc, 1)), uo=UnityOracleBanned(cfg.to_dict(), sd, toks))


@gpu
@pytest.mark.parametrize("tiles", [False, True])
def test_search_with_bans_is_bit_exact_on_oracle_logits(tiny_v2, tiles):
    """Bans chosen from the unbanned winner so that they bite: its first token (n = 1), a later bigram, a trigram that
    starts in the prompt, and [last token, EOS] on the forced-EOS step (min_seq_len = max_len - 2).  Parents, tokens
    and finished hypotheses equal the oracle's at every step (on the forced step, rows whose every candidate is -inf
    finish nothing, and their continuation is not compared)."""
    cfg, uo, eng = tiny_v2["cfg"], tiny_v2["uo"], tiny_v2["model"].engine
    prefix = [cfg.text_eos, tiny_v2["toks"][0].lang_index("spa")]
    torch.manual_seed(5)
    enc = torch.randn(1, 12, cfg.model_dim)
    ML = 24
    for min_len in (1, ML - 2):
        with torch.inference_mode():
            w = uo.beam_search(enc, None, prefix, beam=5, hard_max=ML, min_seq_len=min_len)[0][0][1]
            banned = [[w[2]], [w[4], w[5]], [prefix[1], w[3], w[4]]]
            w = uo.beam_search(enc, None, prefix, beam=5, hard_max=ML, min_seq_len=min_len, banned=banned)[0][0][1]
            banned.append([w[-2], cfg.text_eos] if min_len > 1 else [w[5], w[6], w[7]])
            trace = {"sentence": 0}
            got_o = uo.beam_search(enc, None, prefix, beam=5, hard_max=ML, min_seq_len=min_len, trace=trace, banned=banned)[0]
        assert got_o and got_o[0][1] != w
        decisions, finished = _replay_with_bans(eng, trace, prefix, 5, cfg.text_vocab, banned, min_len, tiles)
        assert len(decisions) == len(trace["beam_idx"])
        for s, (parents, toks, sc) in enumerate(decisions):
            live = [i for i in range(5) if sc[i] != -math.inf]
            assert [parents[i] for i in live] == [trace["beam_idx"][s][i].item() for i in live], f"step {s}: parents differ"
            if s + 1 < len(trace["inputs"]):
                assert [toks[i] for i in live] == [trace["inputs"][s + 1][i].item() for i in live], f"step {s}: tokens differ"
        assert [f[1] for f in finished] == [f[1] for f in trace["finished"]]
        assert all(abs(a[0] - b[0]) < 1e-5 for a, b in zip(finished, trace["finished"]))
        if min_len > 1:
            assert all(f[1][-2] != w[-2] for f in finished)  # the forced EOS was banned after that token


@gpu
def test_engine_search_with_bans_matches_oracle_and_leaves_unbanned_search_alone(tiny_v2):
    """engine.beam_search(banned=...) through the captured ban graph equals the oracle's banned search on the same
    encoder output, launches one kernel more per step, and a later unbanned search on the same state equals the first."""
    from seamless_communication_b200.ops import Seq
    cfg, uo, eng = tiny_v2["cfg"], tiny_v2["uo"], tiny_v2["model"].engine
    prefix = [cfg.text_eos, tiny_v2["toks"][0].lang_index("spa")]
    torch.manual_seed(9)
    enc = torch.randn(2, 16, cfg.model_dim).half().float()
    e = Seq(2, 16, cfg.model_dim, buf=enc.to(dev).half().reshape(-1, cfg.model_dim).contiguous())
    plain = eng.beam_search(e, None, prefix, beam=5, hard_max=20)
    w = plain[0][0][1]
    banned = [[w[2]], [w[3], w[4]]]
    k0 = eng.graph_kernels
    got = eng.beam_search(e, None, prefix, beam=5, hard_max=20, banned=banned)
    with torch.inference_mode():
        ref = uo.beam_search(enc, None, prefix, beam=5, hard_max=20, banned=banned)
    for b in range(2):
        assert got[b][0][1] == ref[b][0][1] or abs(got[b][0][0] - ref[b][0][0]) < 2e-2
        for _, ids in got[b]:
            for s in banned:
                n = len(s)
                assert all(ids[t - n + 1:t + 1] != s for t in range(len(prefix), len(ids)))
    assert got[0][0][1] != w
    assert eng.graph_kernels > k0
    again = eng.beam_search(e, None, prefix, beam=5, hard_max=20)
    assert again == plain
    key = [k for k, st in eng._graphs.items() if st.get("g_sel_ban") is not None]
    st = eng._graphs[key[0]]
    assert st["n_sel_ban"] == st["n_sel"] + 1


# ------------------------------------------------------------------------------------------------ GPU: end to end
def _words_of(tok, hyp, P):
    """Words of a hypothesis that are whole "▁" pieces (the next piece starts a new word or ends the text)."""
    pieces = [tok.model.index_to_token(int(i)) for i in hyp]
    out = []
    for t in range(P, len(hyp) - 1):
        nxt = pieces[t + 1]
        if pieces[t].startswith(S.SPACE) and len(pieces[t]) > 1 and (nxt.startswith(S.SPACE) or t + 1 == len(hyp) - 1):
            out.append(pieces[t][1:])
    return out


def _checker(tmp_path, tgt_words, src_words=("zzzzqq",)):
    import codecs
    from seamless_communication_b200.toxicity import load_etox_bad_word_checker
    d = tmp_path / "etox"
    d.mkdir(exist_ok=True)
    (d / "spa_twl.txt").write_text("".join(codecs.encode(w, "rot_13") + "\n" for w in tgt_words), encoding="utf-8")
    (d / "eng_twl.txt").write_text("".join(codecs.encode(w, "rot_13") + "\n" for w in src_words), encoding="utf-8")
    return load_etox_bad_word_checker("mintox", dataset_dir=str(d))


def _contains(ids, seq, P):
    n = len(seq)
    return any(ids[t - n + 1:t + 1] == seq for t in range(P, len(ids)) if t - n + 1 >= 0)


def _run_e2e(tmp_path, monkeypatch, model, voc, toks, task, v1):
    from seamless_communication_b200.inference import Translator
    from seamless_communication_b200.nn import get_seqs_and_padding_mask
    from seamless_communication_b200.toxicity.mintox import _extract_bad_words_with_batch_indices, banned_sequence_processor
    tok = toks[0]
    P = 2
    opts = SequenceGeneratorOptions(hard_max_seq_len=20)
    uopts = SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40)
    plain = Translator(model, voc, device="cuda:0")
    waves = S.make_waveforms(4, 32000, seed=31)
    src = plain.fbank_batch(waves)
    texts0, speech0 = plain.predict(src, task, "spa", text_generation_opts=opts, unit_generation_opts=uopts)
    hyps0 = [h[0][1] for h in Translator._tls.generator.last_text_output.hypotheses]
    # the word lists: a word of row 0 and a word pair of row 2 (as one entry) are added toxicity
    w0, w2 = _words_of(tok, hyps0[0], P), _words_of(tok, hyps0[2], P)
    assert w0 and len(w2) >= 2
    tgt_words = [w0[0], w2[0] + " " + w2[1]]
    checker = _checker(tmp_path, tgt_words)
    words, rows = _extract_bad_words_with_batch_indices(texts0, texts0, "eng", "spa", checker)
    assert 0 in rows and 2 in rows and len(rows) < 4
    proc = banned_sequence_processor(tok, list(dict.fromkeys(words)))
    seqs, mask = get_seqs_and_padding_mask(src)
    idx = torch.tensor(rows, device=dev)
    ut = plain.unit_tokenizer if task == "s2st" else None
    from seamless_communication_b200.inference.translator import Modality
    out_mod = Modality.SPEECH if task == "s2st" else Modality.TEXT
    before = Translator.get_prediction(model, tok, ut, seqs[idx], None, Modality.SPEECH, out_mod, "spa", opts, uopts)
    mt = Translator(model, voc, device="cuda:0", apply_mintox=True, bad_word_checker=checker)
    texts, speech = mt.predict(src, task, "spa", src_lang="eng", text_generation_opts=opts, unit_generation_opts=uopts)
    assert opts.step_processor is None  # the caller's options are not mutated
    new_hyps = [h[0][1] for h in Translator._tls.generator.last_text_output.hypotheses]
    gen_alone = SequenceGeneratorOptions(hard_max_seq_len=20, step_processor=proc)
    alone_texts, alone_units = Translator.get_prediction(model, tok, ut, seqs[idx], None, Modality.SPEECH, out_mod, "spa",
                                                         gen_alone, uopts)
    alone_gen = Translator._tls.generator
    assert [h[0][1] for h in alone_gen.last_text_output.hypotheses] == new_hyps
    for j, i in enumerate(rows):
        assert texts[i] == alone_texts[j]
        for s in proc.banned_seqs:
            assert not _contains(new_hyps[j], s, P), (i, s)
    assert any(texts[i] != texts0[i] for i in rows)
    for i in range(4):
        if i not in rows:
            assert texts[i] == texts0[i]
    if task == "s2st":
        pad = 1
        for i in range(4):
            if i not in rows:
                assert speech.units[i] == speech0.units[i]
                if v1:
                    assert torch.equal(speech.audio_wavs[i], speech0.audio_wavs[i])
        if not v1:
            for j, i in enumerate(rows):
                assert speech.units[i] == [u for u in alone_units[j].tolist() if u != pad]
    # an unbanned search after the banned one, on the same cached state, is the unbanned search
    after = Translator.get_prediction(model, tok, ut, seqs[idx], None, Modality.SPEECH, out_mod, "spa", opts, uopts)
    assert after[0] == before[0]
    # nothing flagged: bit-identical outputs and no second search
    calls = []
    orig = Translator.get_prediction.__func__
    monkeypatch.setattr(Translator, "get_prediction", classmethod(lambda cls, *a, **k: calls.append(1) or orig(cls, *a, **k)))
    quiet = Translator(model, voc, device="cuda:0", apply_mintox=True, bad_word_checker=_checker(tmp_path, ["zzzzzz"]))
    texts_q, speech_q = quiet.predict(src, task, "spa", src_lang="eng", text_generation_opts=opts, unit_generation_opts=uopts)
    assert len(calls) == 1 and texts_q == texts0
    if task == "s2st":
        assert speech_q.units == speech0.units
        assert all(torch.equal(a, b) for a, b in zip(speech_q.audio_wavs, speech0.audio_wavs))


@gpu
@pytest.mark.parametrize("task", ["s2st", "s2tt"])
def test_mintox_end_to_end_tiny_v2(tiny_v2, tmp_path, monkeypatch, task):
    _run_e2e(tmp_path, monkeypatch, tiny_v2["model"], tiny_v2["voc"], tiny_v2["toks"], task, v1=False)


@gpu
def test_asr_returns_the_s2tt_texts(tiny_v2):
    """MinTox takes the first pass's texts as its source texts: the reference's predict(x, "ASR", tgt_lang) is the same
    search over the same input."""
    from seamless_communication_b200.inference import Translator
    tr = Translator(tiny_v2["model"], tiny_v2["voc"], device="cuda:0")
    src = tr.fbank_batch(S.make_waveforms(3, 32000, seed=8))
    opts = SequenceGeneratorOptions(hard_max_seq_len=20)
    assert tr.predict(src, "asr", "spa", text_generation_opts=opts)[0] == tr.predict(src, "s2tt", "spa", text_generation_opts=opts)[0]


@gpu
def test_mintox_end_to_end_tiny_v1(tmp_path, monkeypatch):
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    cfg, vc = C.tiny_v1(), C.tiny_vocoder()
    sd = S.make_unity_state_dict(cfg, 0, dec_gain=4.0, with_t2u=True)
    e = sd["t2u_model.final_proj.weight"].clone()  # a reachable unit EOS, as test_v1_s2st.with_reachable_eos
    g = torch.Generator().manual_seed(11)
    e[cfg.unit_eos] = (torch.randn(cfg.model_dim, generator=g) * 0.75 * cfg.model_dim ** -0.5).half().float()
    sd = {**sd, "t2u_model.final_proj.weight": e, "t2u_model.decoder_frontend.embed.weight": e}
    toks = S.make_tokenizers(cfg)
    model = load_unity_model("tiny_v1", state_dict=sd, tokenizers=toks)
    voc = load_vocoder_model("tiny", state_dict=S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True))
    _run_e2e(tmp_path, monkeypatch, model, voc, toks, "s2st", v1=True)
