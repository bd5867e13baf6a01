"""Transcriber (inference/transcriber.py): the timestamp restatement against the reference's own functions
(tests/golden/transcriber.json), the API's refusals, and on the GPU both new kernels, the search's per-hypothesis scores
and the whole path against the CPU oracle (tests/oracle_transcriber.py)."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle_transcriber import (UnityOracleTranscriber, lis, random_attention, start_bins, start_bins_from_rows,  # noqa: E402
                                word_stats)

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
dev = "cuda"


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(G, "transcriber.json")) as f:
        return json.load(f)


# ------------------------------------------------------------------------------------------------ CPU
def test_restatement_matches_reference_timestamps(golden):
    for c in golden["timestamps"]:
        rows = np.array(c["rows"], dtype=np.float32)
        bins = start_bins_from_rows(rows, c["width"])
        assert bins == c["bins"], (c["name"], c["width"])
        F = rows.shape[1] - 2
        assert [3.7 / F * b for b in bins] == c["times_3_7s"]
    for c in golden["random"]:
        bins = start_bins_from_rows(random_attention(c["seed"], c["n"], c["S"]), c["width"])
        assert bins == c["bins"], (c["seed"], c["width"])
        assert [3.7 / (c["S"] - 2) * b for b in bins] == c["times_3_7s"]


def test_restatement_matches_reference_lis(golden):
    for c in golden["lis"]:
        arr = c["arr"]
        L, prev, i = lis([a for a, _ in arr])
        path = [i]
        while prev[i] != i:
            i = prev[i]
            path.append(i)
        assert max(L) == c["max"] and [arr[j] for j in reversed(path)] == c["seq"]


def test_word_grouping_matches_reference(golden):
    from seamless_communication_b200.inference import Transcriber
    for c in golden["words"]:
        want = [tuple(w) for w in c["out"]]
        assert word_stats(c["pieces"], c["times"], c["scores"]) == want
        got = Transcriber._collect_word_level_stats(c["pieces"], c["times"], c["scores"])
        assert [(t.text, t.time_s, t.prob) for t in got] == want


def test_zero_column_normalises_to_zero():
    A = np.array([[0.0, 1.0, 0.0], [0.0, 3.0, 2.0]])
    assert start_bins(A, 1) == [0, 1]


def test_api_refusals():
    from seamless_communication_b200.inference import Transcriber
    t = Transcriber.__new__(Transcriber)  # the checks run before any device work
    wav = torch.zeros(16000)
    with pytest.raises(ValueError, match="odd"):
        t.transcribe(wav, "eng", filter_width=4)
    with pytest.raises(ValueError, match="odd"):
        t.transcribe_batch([wav], "eng", filter_width=0)
    with pytest.raises(ValueError, match="above 7"):
        t.transcribe(wav, "eng", filter_width=9)
    with pytest.raises(ValueError, match="chunk_size_sec"):
        t.transcribe(torch.zeros(16000 * 21), "eng")
    with pytest.raises(ValueError, match="longer than 20 s"):
        t.transcribe_batch([wav, torch.zeros(16000 * 21)], "eng")
    with pytest.raises(NotImplementedError, match="Demucs"):
        t.transcribe(wav, "eng", denoise=True)
    with pytest.raises(ValueError, match="sample_rate"):
        t.transcribe(wav, "eng", sample_rate=8000)
    with pytest.raises(ValueError, match="one channel"):
        t.transcribe(torch.zeros(16000, 2), "eng")
    with pytest.raises(TypeError, match="temperature"):
        t.transcribe(wav, "eng", temperature=0.5)
    with pytest.raises(TypeError, match="step_processor"):
        t.transcribe_batch([wav], "eng", step_processor=None, beam_size=2)


# ------------------------------------------------------------------------------------------------ GPU: kernels
@pytest.mark.gpu
@pytest.mark.parametrize("s_enc,beam,splits", [(1, 1, 1), (2, 5, 2), (31, 1, 3), (32, 5, 4), (33, 1, 5), (63, 5, 6),
                                               (64, 1, 7), (65, 5, 8), (127, 1, 8), (128, 5, 1), (129, 1, 2), (752, 5, 3)])
def test_cross_attn_weights_kernel_against_float64(s_enc, beam, splits):
    """hist[step][r][t] = sum_h softmax(q_h . k_h / 8)[t] against float64 from the same partials.  Bound: q is the fp16
    rounding of the fp32 partial sum (|dq| <= 2^-11 |q| + splits 2^-24 sum|partials|), so each score moves by at most
    d_h = sum_d |dq_d||k_d| / 8 + fp32 dot rounding; a softmax weight then moves by at most p (e^{2 d_h} - 1), plus fp32
    rounding of exp / sum / division (8 ulp per head)."""
    from seamless_communication_b200 import _lib, ops
    torch.manual_seed(s_enc * 10 + beam)
    H, M, B = 4, 256, 3
    R = B * beam
    SR = ops.slice_rows(R)
    part = torch.randn(splits, SR, M, device=dev) * (0.6 / math.sqrt(splits))
    bias = torch.randn(M, device=dev) * 0.1
    kv = torch.randn(B * s_enc, 2 * M, device=dev).half()
    lens = torch.tensor([s_enc, max(1, s_enc - 7), max(1, s_enc // 2)], dtype=torch.int32, device=dev)
    kv3 = kv.view(B, s_enc, 2 * M)
    for b in range(B):
        kv3[b, int(lens[b]):, :M] = float("nan")  # never read
    ML, step = 4, 2
    hist = torch.full((ML, R, s_enc), -7.0, device=dev)
    step_t = torch.tensor([step], dtype=torch.int32, device=dev)
    ops.decode_cross_attn_weights(part.view(-1, M), splits, SR, bias, kv, lens, s_enc, step_t, hist, R, beam, H)
    torch.cuda.synchronize()
    h = hist.cpu()
    assert (h[torch.arange(ML) != step] == -7.0).all()  # only the *step_ptr slab is written
    p64 = part[:, :R].double().sum(0).cpu() + bias.double().cpu()
    q16 = (part[:, :R].sum(0) + bias).half().double().cpu()
    k64 = kv3[:, :, :M].double().cpu()
    for r in range(R):
        b = r // beam
        n = int(lens[b])
        got = h[step, r]
        assert (got[n:] == 0).all()
        want = torch.zeros(n, dtype=torch.float64)
        bound = torch.zeros(n, dtype=torch.float64)
        for hh in range(H):
            sl = slice(hh * 64, hh * 64 + 64)
            kk = k64[b, :n, sl]
            s = kk @ p64[r, sl] / 8
            p = torch.softmax(s, 0)
            dq = p64[r, sl].abs() * 2.0 ** -11 + splits * 2.0 ** -24 * part[:, r, sl].abs().sum(0).double().cpu() + 2.0 ** -24
            d = (kk.abs() @ dq) / 8 + 64 * 2.0 ** -24 * (kk.abs() @ q16[r, sl].abs()) / 8
            want += p
            bound += p * torch.expm1(2 * d.max()) + 8 * 2.0 ** -24 * (p + 1e-30)
        err = (got[:n].double() - want).abs()
        assert bool((err <= bound + H * 2.0 ** -22).all()), (r, float((err - bound).max()))


def _nan_hist(rows_per_pos, slots, P, n, F, S, ML, R):
    """hist full of NaN except the entries a gather reads: positions P-1 .. P+n-2 at the row's slots, frames 1 .. F."""
    hist = torch.full((ML, R, S), float("nan"))
    for k in range(n):
        t = P - 1 + k
        hist[t, slots[t], 1:1 + F] = torch.from_numpy(rows_per_pos[k, 1:1 + F])
    return hist


@pytest.mark.gpu
def test_token_timestamps_kernel_bit_exact(golden):
    """sb_token_timestamps equals the float64 restatement on the fixture matrices, on random ones up to n = 1024
    positions and F = 4096 frames, and on one with zero-sum columns (normalised to 0), reading nothing but the winner's
    entries (everything else is NaN)."""
    from seamless_communication_b200 import ops
    cases = [(np.array(c["rows"], dtype=np.float32), c["width"]) for c in golden["timestamps"]]
    cases += [(random_attention(c["seed"], c["n"], c["S"]), c["width"]) for c in golden["random"]]
    cases += [(random_attention(90, 1021, 130), 3), (random_attention(91, 40, 4098), 3), (random_attention(92, 300, 700), 5),
              (random_attention(93, 64, 126), 7), (random_attention(94, 12, 126), 1)]
    zero = random_attention(95, 30, 50)
    zero[1:, [1, 7, 20, 48]] = 0.0  # A's columns 0, 6, 19 and F-1 sum to 0 and normalise to 0
    cases += [(zero, 1), (zero, 3), (zero, 7)]
    P, R, g = 2, 3, torch.Generator().manual_seed(3)
    for rows, w in cases:
        n, S = rows.shape[0] - 1, rows.shape[1]
        F, ML = S - 2, P + n + 1
        slots = torch.randint(0, R, (ML,), generator=g, dtype=torch.int32)
        hist = _nan_hist(rows[1:], slots, P, n, F, S, ML, R)
        starts = ops.token_timestamps(hist.to(dev), slots[None].to(dev), torch.tensor([n], dtype=torch.int32, device=dev),
                                      None, P, w).cpu()
        assert starts[0].tolist() == start_bins_from_rows(rows, w), (n, S, w)


@pytest.mark.gpu
def test_token_timestamps_ragged_batch_and_limits():
    """Rows of one batch with their own n and encoder length equal each row alone; n = 0 and F < 1 rows write nothing;
    the refusals come before any launch."""
    from seamless_communication_b200 import _lib, ops
    P, R, S, ML = 2, 4, 40, 60
    g = torch.Generator().manual_seed(5)
    ns, lens = [17, 0, 5, 30], [40, 33, 2, 3]
    slots = torch.randint(0, R, (4, ML), generator=g, dtype=torch.int32)
    hist = torch.full((ML, R, S), float("nan"))
    want = []
    for b in range(4):
        rows = random_attention(200 + b, ns[b], lens[b])
        F = lens[b] - 2
        for k in range(ns[b]):
            if F >= 1:
                hist[P - 1 + k, slots[b, P - 1 + k], 1:1 + F] = torch.from_numpy(rows[1 + k, 1:1 + F])
        want.append(start_bins_from_rows(rows, 3) if ns[b] and F >= 1 else [0] * ns[b])
    starts = ops.token_timestamps(hist.to(dev), slots.to(dev), torch.tensor(ns, dtype=torch.int32, device=dev),
                                  torch.tensor(lens, dtype=torch.int32, device=dev), P, 3).cpu()
    for b in range(4):
        assert starts[b, :ns[b]].tolist() == want[b]
    with pytest.raises(RuntimeError, match="above 7"):
        ops.token_timestamps(hist.to(dev), slots.to(dev), torch.tensor(ns, dtype=torch.int32, device=dev), None, P, 9)
    with pytest.raises(RuntimeError, match="odd"):
        ops.token_timestamps(hist.to(dev), slots.to(dev), torch.tensor(ns, dtype=torch.int32, device=dev), None, P, 2)
    big = torch.zeros((3, 1, 4099), device=dev)
    with pytest.raises(RuntimeError, match="above 4096"):
        ops.token_timestamps(big, torch.zeros((1, 3), dtype=torch.int32, device=dev), torch.ones(1, dtype=torch.int32, device=dev),
                             None, 1, 3)


# ------------------------------------------------------------------------------------------------ GPU: search and path
def with_reachable_text_eos(sd, cfg, scale=0.5, seed=11):
    """The synthetic text decoder rarely scores EOS; a larger EOS row (tied embedding / projection) ends searches early
    and at different lengths (on the inputs below: 12, 12 and 87 tokens of a 144-token budget at beam 1)."""
    e = sd["final_proj.weight"].clone()
    g = torch.Generator().manual_seed(seed)
    e[cfg.text_eos] = (torch.randn(cfg.model_dim, generator=g) * scale * cfg.model_dim ** -0.5).half().float()
    return {**sd, "final_proj.weight": e, "text_decoder_frontend.embed.weight": e}


def _tiny(arch):
    from seamless_communication_b200 import config as C, synthetic as S
    from seamless_communication_b200.inference import Transcriber
    cfg = getattr(C, arch)()
    sd = with_reachable_text_eos(S.make_unity_state_dict(cfg, 0, dec_gain=4.0), cfg)
    toks = S.make_tokenizers(cfg)
    tr = Transcriber(arch, "cuda", state_dict=sd, tokenizer=toks)
    if cfg.encoder_variant == "v1":
        from oracle_v1 import UnityOracleV1

        class OracleV1(UnityOracleTranscriber, UnityOracleV1):
            pass
        cls = OracleV1
    else:
        cls = UnityOracleTranscriber
    uo = cls(cfg.to_dict(), sd, toks)
    uo.layer0 = cls(cfg.to_dict(), sd, toks, record_layer=0)  # the first layer's attention: a negative control
    return cfg, toks, tr, uo


@pytest.fixture(scope="module")
def tiny_v2():
    return _tiny("tiny_v2")


@pytest.fixture(scope="module")
def tiny_v1():
    return _tiny("tiny_v1")


# The recorded attention (head-summed, so each row sums to the number of heads, here 2) against the fp32 oracle's: the
# engine stores the encoder output, the cross K/V and every decoder activation in fp16 and runs its GEMMs on fp16 inputs,
# so each attention score carries the fp16 rounding of q and K (relative 2^-11 each) propagated through two decoder
# layers.  Score errors of up to 2.5e-3 move a weight p by at most p (e^{2 * 2.5e-3} - 1) < 5e-3 p, i.e. at most 1e-2
# over a head-summed row: the bound.  Measured on an H100: see DESIGN.md section 13.  Its discriminating power is
# checked in the same test: the oracle's rows one position earlier or later, and the first layer's attention, are all
# further than the bound from the device's rows.
ATTN_BOUND = 1e-2


def _filtered(A, width):
    n, F = A.shape
    s = A.sum(0)
    A = np.where(s != 0, A / np.where(s != 0, s, 1.0), 0.0)
    r = width // 2
    pad = np.zeros((n + 2 * r, F + 2 * r))
    pad[r:r + n, r:r + F] = A
    return np.sort(np.lib.stride_tricks.sliding_window_view(pad, (width, width)).reshape(n, F, -1), -1)[:, :, width * width // 2]


def _filtered_bound(A, e, width):
    """Per element, how far the filtered value of a matrix within e (elementwise) of A can be from A's: the column
    normalisation x / s moves by at most (e + (x / s) n e) / (s - n e), and a median moves by at most the largest
    movement in its window (zero padding does not move)."""
    n, F = A.shape
    s = A.sum(0)
    assert (s > n * e).all(), "a column is too small for the attention bound to bound its normalisation"
    bn = (e + (A / s) * n * e) / (s - n * e)
    r = width // 2
    pad = np.zeros((n + 2 * r, F + 2 * r))
    pad[r:r + n, r:r + F] = bn
    return np.lib.stride_tricks.sliding_window_view(pad, (width, width)).reshape(n, F, -1).max(-1)


def _audit(bins_dev, A_dev, bins_or, A_or, width, what):
    """Start bins of the device path against the oracle's.  The kernel's bins equal the restatement on the device's own
    attention bit for bit, and that attention is within ATTN_BOUND of the oracle's.  Where the bins part, every column
    whose argmax differs must be a near-tie that the bound explains: the oracle's filtered values of the two rows differ
    by at most the sum of their propagated bounds."""
    assert bins_dev == start_bins(A_dev, width), what
    err = np.abs(A_dev - A_or).max()
    assert err <= ATTN_BOUND, f"{what}: recorded attention {err:.3e} from the oracle's"
    if bins_dev == bins_or:
        return
    fd, fo = _filtered(A_dev, width), _filtered(A_or, width)
    bf = _filtered_bound(A_or, ATTN_BOUND, width)
    cd, co = fd.argmax(0), fo.argmax(0)
    diff = np.nonzero(cd != co)[0]
    assert len(diff) > 0, f"{what}: same column maxima but different start bins"
    for j in diff:
        assert fo[co[j], j] - fo[cd[j], j] <= bf[co[j], j] + bf[cd[j], j], f"{what}: column {j} is not a near-tie"


def _expected_words(pieces, seconds, F, bins, scores):
    per_bin = seconds / F if F >= 1 else 0.0
    return word_stats(pieces, [per_bin * b for b in bins], scores)


def _same_words(got, want, prob_tol, what):
    """Words equal in text and start time; probabilities within prob_tol relative (exp of scores within a tolerance)."""
    assert [(t.text, t.time_s) for t in got] == [(w[0], w[1]) for w in want], what
    for t, w in zip(got, want):
        assert abs(t.prob - w[2]) <= prob_tol * max(t.prob, w[2]) + 1e-15, (what, t, w)


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ["tiny_v2", "tiny_v1"])
@pytest.mark.parametrize("beam", [1, 5])
def test_transcribe_against_oracle(arch, beam, request):
    """Tokens equal the oracle's (at most one of the three searches may part from it, at an audited near-tie of the search
    itself).  Where tokens agree: the recorded attention within ATTN_BOUND of the oracle's (and further than that from
    its neighbouring positions and from the first layer), start bins equal up to near-ties the bound explains, per-token
    scores within 2e-2 (fp16 storage against the fp32 oracle), and the returned words equal the oracle's word grouping
    in text and start time, their probabilities within the scores' tolerance."""
    from oracle.unity_oracle import fbank as o_fbank
    from seamless_communication_b200 import synthetic as S
    cfg, toks, tr, uo = request.getfixturevalue(arch)
    waves = S.make_waveforms(3, 48000, seed=5)
    prefix = [cfg.text_eos, toks[0].lang_index("eng")]
    diverged = 0
    for i, w in enumerate(waves):
        t = tr.transcribe(w, "eng", beam_size=beam)
        A_dev, n_dev = tr.engine.harvest_attention()
        stamps = tr.engine.token_timestamps(3)[0]
        st = tr.engine._last_search_state
        j = st["best_fin"][0]
        ids = st["fin"]["seqs"][0, j, :int(st["fin"]["len"][0, j])].tolist()[len(prefix):-1]
        fb = o_fbank(w)
        fb = fb[:fb.shape[0] - fb.shape[0] % 2][None]
        ref = uo.transcribe(fb, None, [w.numel() / 16000], prefix, width=3, beam=beam)[0]
        what = f"{arch} beam {beam} row {i}"
        assert n_dev[0] == len(ids) and len(t.tokens) <= len(ids) and (len(ids) == 0) == (len(t.tokens) == 0), what
        F = ref["F"]
        A = A_dev[0, :len(ids), 1:1 + F].double().cpu().numpy()
        if ids:
            assert stamps[0] == start_bins(A, 3), what  # the kernel on the device's own attention, bit for bit
        if ids != ref["ids"]:
            # an fp16-vs-fp32 near-tie of the search (as smoke() allows): the device's hypothesis, scored by the oracle, is
            # within 2e-2 of the oracle's own best score; timestamps are then compared on the matching searches only
            diverged += 1
            full = torch.tensor(prefix + ids + [cfg.text_eos])[None]
            enc, _ = uo.encode_speech(fb, None)
            lp = torch.log_softmax(uo.project(uo.decoder(uo.embed_text(full[:, :-1], 0), enc, None)).float(), -1)[0]
            sc = sum(float(lp[k, full[0, k + 1]]) for k in range(full.shape[1] - 1)) / (full.shape[1] - 1)
            assert abs(sc - uo.records[0][0]["score"]) < 2e-2, what
            continue
        if F >= 1 and ids:
            _audit(stamps[0], A, ref["bins"], ref["A"], 3, what)
            # negative controls: a position off by one either way, or another layer, would not pass the bound
            P, n = len(prefix), len(ids)
            at = ref["attn"].numpy()
            for lo in (P - 2, P):
                if at.shape[0] >= lo + n:
                    assert np.abs(A - at[lo:lo + n, 1:1 + F]).max() > ATTN_BOUND, what
            ref0 = uo.layer0.transcribe(fb, None, [w.numel() / 16000], prefix, width=3, beam=beam)[0]
            assert ref0["ids"] == ids and np.abs(A - ref0["A"]).max() > ATTN_BOUND, what
        assert np.allclose(stamps[1], ref["scores"], rtol=0, atol=2e-2)
        # the public output: words from the oracle's pieces and scores at the device's (audited) bins
        pieces = [toks[0].model.index_to_token(x) for x in ids]
        if stamps[0] == ref["bins"]:
            assert _expected_words(pieces, w.numel() / 16000, F, stamps[0], ref["scores"]) == \
                word_stats(pieces, ref["times"], ref["scores"])
        _same_words(t.tokens, _expected_words(pieces, w.numel() / 16000, F, stamps[0], ref["scores"]), math.expm1(2e-2), what)
    assert diverged <= 1, f"{arch} beam {beam}: {diverged} of 3 searches part from the oracle's"


@pytest.mark.gpu
def test_fin_scores_bit_exact_on_oracle_logits(tiny_v2):
    """Driving the select half of the search with the oracle's fp32 logits (as test_gpu_parity's harness does), every
    finished hypothesis's fin_scores hold its parent row's cumulative scores bit for bit and its EOS score last, and equal
    the oracle's cumulative scores of the same hypothesis within the harness's 1e-5."""
    import ctypes as Ct
    from oracle.unity_oracle import fbank as o_fbank
    from seamless_communication_b200 import _lib, synthetic as S
    from seamless_communication_b200._lib import BeamDesc, check
    cfg, toks, tr, uo = tiny_v2
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    prefix = [cfg.text_eos, toks[0].lang_index("eng")]
    w = S.make_waveforms(1, 48000, seed=5)[0]
    fb = o_fbank(w)[None]
    enc, lens = uo.encode_speech(fb, None)
    trace = {"sentence": 0}
    beam = 5
    uo.beam_search(enc, None, prefix, beam=beam, soft_max=(1, 40), trace=trace)
    V, ML, P, R = cfg.text_vocab, trace["max_len"], len(prefix), beam
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
    fin = dict(count=torch.zeros(1, **i32), score=torch.full((1, beam), -math.inf, device=dev), len=torch.zeros((1, beam), **i32),
               seqs=torch.zeros((1, beam, ML), **i32), active=torch.ones(1, **i32), n_active=torch.ones(1, **i32),
               anc=torch.zeros((1, beam, ML), **i32), scores=torch.full((1, beam, ML), float("nan"), device=dev))
    d = BeamDesc()
    d.batch, d.beam, d.max_len, d.vocab, d.K = 1, beam, ML, V, K
    d.step_ptr, d.prefix_len, d.eos_idx, d.min_len, d.len_penalty = step.data_ptr(), P, cfg.text_eos, 1, 1.0
    d.cand_val, d.cand_idx, d.eos_lprob = cv.data_ptr(), ci.data_ptr(), el.data_ptr()
    d.seqs, d.scores, d.anc = seqs.data_ptr(), scores.data_ptr(), anc.data_ptr()
    d.fin_count, d.fin_score, d.fin_len = fin["count"].data_ptr(), fin["score"].data_ptr(), fin["len"].data_ptr()
    d.fin_seqs, d.active, d.n_active, d.fin_anc = fin["seqs"].data_ptr(), fin["active"].data_ptr(), fin["n_active"].data_ptr(), fin["anc"].data_ptr()
    d.fin_scores = fin["scores"].data_ptr()
    snaps = {}
    for s_i, lg in enumerate(trace["logits"]):
        logits[:, :V] = lg.to(dev)
        check(lib.sb_logits_topk(logits.data_ptr(), ld, R, V, cfg.text_pad, cfg.text_eos, cfg.text_unk, 0.0, K, cv.data_ptr(),
                                 ci.data_ptr(), el.data_ptr(), st))
        snaps[P - 1 + s_i] = (scores.cpu().clone(), el.cpu().clone())
        check(lib.sb_beam_step(Ct.byref(d), st))
        check(lib.sb_step_advance(step.data_ptr(), st))
        if int(fin["active"].item()) == 0:
            break
    n = int(fin["count"].item())
    assert n >= 2
    want = {tuple(r["ids"]): r["cum"] for r in uo.records[0]}
    for j in range(n):
        L = int(fin["len"][0, j])
        ids = tuple(fin["seqs"][0, j, :L].tolist())
        got = fin["scores"][0, j, :L].cpu()
        s_fin = L - 2
        row = int(fin["anc"][0, j, s_fin])
        sc, eos_lp = snaps[s_fin]
        # bit for bit: the parent row's cumulative scores, then the fp32 sum that scored its EOS
        assert torch.equal(got[:L - 1], sc[row, :L - 1]), j
        assert got[L - 1].item() == (sc[row, s_fin] + eos_lp[row]).item(), j
        assert torch.isnan(fin["scores"][0, j, L:]).all()
        # and the oracle's cumulative scores up to the fp32 log-sum-exp order (the harness's own 1e-5)
        assert torch.allclose(got, want[ids], rtol=0, atol=1e-5), j


def _winner_ids(eng, b, P):
    st = eng._last_search_state
    j = st["best_fin"][b]
    return st["fin"]["seqs"][b, j, :int(st["fin"]["len"][b, j])].tolist()[P:-1] if j >= 0 else []


def _step_gap(uo, fb, prefix, a, b):
    """Oracle lprob gap, on the input alone, between the two tokens at the first position where hypotheses a and b part."""
    k = next(i for i in range(min(len(a), len(b)) + 1) if i == len(a) or i == len(b) or a[i] != b[i])
    eos = uo.c["text_eos"]
    ta, tb = (a + [eos])[k], (b + [eos])[k]
    ids = torch.tensor(prefix + a[:k])[None]
    enc, _ = uo.encode_speech(fb, None)
    lp = torch.log_softmax(uo.project(uo.decoder(uo.embed_text(ids, 0), enc, None)).float(), -1)[0, -1]
    return abs(float(lp[ta] - lp[tb]))


@pytest.mark.gpu
def test_transcribe_batch_equals_rows_alone(tiny_v2):
    """A ragged list through one search equals each row transcribed alone: tokens equal, the recorded attention within
    ATTN_BOUND, start bins equal up to near-ties the bound explains, scores within 2e-2, and word times computed from the
    row's own duration and frame count (equal to the row alone's wherever the bins are).  The encoder of a padded row reads the padding frames the adaptor's
    strided conv reaches, so a search may part from the row alone at most once in the list, and only at a near-tie
    decision: at the first position where the hypotheses part, the oracle's lprobs of the two tokens (on the row alone) are
    within 5e-2 (fp16 rounding plus the padding frames' effect on the encoder)."""
    from oracle.unity_oracle import fbank as o_fbank
    from seamless_communication_b200 import synthetic as S
    cfg, toks, tr, uo = tiny_v2
    P = 2
    prefix = [cfg.text_eos, toks[0].lang_index("eng")]
    full = S.make_waveforms(3, 48000, seed=5)
    waves = [full[0], full[1, :40000], full[2, :31000]]
    batch = tr.transcribe_batch(waves, "eng")
    A_b, n_b = tr.engine.harvest_attention()
    lens_b = tr.engine._last_search_state["enc_lens"].tolist()
    stamps_b = tr.engine.token_timestamps(3)
    ids_b = [_winner_ids(tr.engine, i, P) for i in range(3)]
    diverged = 0
    for i, w in enumerate(waves):
        alone = tr.transcribe(w, "eng")
        A_a, n_a = tr.engine.harvest_attention()
        stamps_a = tr.engine.token_timestamps(3)[0]
        ids_a = _winner_ids(tr.engine, 0, P)
        if ids_b[i] != ids_a:
            diverged += 1
            fb = o_fbank(w)
            fb = fb[:fb.shape[0] - fb.shape[0] % 2][None]
            assert _step_gap(uo, fb, prefix, ids_b[i], ids_a) < 5e-2, f"row {i}: not a near-tie"
            continue
        F = int(lens_b[i]) - 2
        assert F == tr.engine._last_search_state["S_enc"] - 2, f"row {i}: the batch row's frame count is not its own"
        if n_a[0] and F >= 1:
            _audit(stamps_b[i][0], A_b[i, :n_b[i], 1:1 + F].double().cpu().numpy(), stamps_a[0],
                   A_a[0, :n_a[0], 1:1 + F].double().cpu().numpy(), 3, f"row {i}")
        assert np.allclose(stamps_b[i][1], stamps_a[1], rtol=0, atol=2e-2)
        # the returned words: the row's own seconds / F per bin, its own bins and scores, exactly
        pieces = [toks[0].model.index_to_token(x) for x in ids_b[i]]
        _same_words(batch[i].tokens, _expected_words(pieces, w.numel() / 16000, F, stamps_b[i][0], stamps_b[i][1]), 0.0,
                    f"row {i}")
        assert [t.text for t in batch[i].tokens] == [t.text for t in alone.tokens] or stamps_b[i][0] != stamps_a[0]
        if stamps_b[i][0] == stamps_a[0]:
            assert [t.time_s for t in batch[i].tokens] == [t.time_s for t in alone.tokens], f"row {i}"
    assert diverged <= 1


@pytest.mark.gpu
def test_translate_after_recording_search_is_unchanged(tiny_v2):
    """A recording search leaves the engine's other searches as they were: same texts, same graph launch count."""
    from seamless_communication_b200 import synthetic as S
    from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator
    cfg, toks, tr, uo = tiny_v2
    waves = S.make_waveforms(2, 48000, seed=8)
    tl = Translator(tr.model, None, "cuda", output_modality=None)
    opts = SequenceGeneratorOptions(beam_size=1, soft_max_seq_len=(1, 128))
    src = tl.fbank_batch(waves)

    def run():
        k0 = tr.engine.graph_kernels
        texts, _ = tl.predict(src, "s2tt", "eng", text_generation_opts=opts)
        torch.cuda.synchronize()
        return texts, tr.engine.graph_kernels - k0
    before = run()
    tr.transcribe_batch(list(waves), "eng")
    assert tr.engine._last_search_state["n_fwd_attn"] == tr.engine._last_search_state["n_fwd"] + 1
    assert run() == before


@pytest.mark.gpu
def test_small_v2_full_width_20s():
    """M = 1024, 16 heads, one 20 s input: start bins of the device path equal the restatement on its own attention, and
    the attention equals a float64 recomputation from the recorded search within the kernel test's bound order."""
    from seamless_communication_b200.inference import Transcriber
    from seamless_communication_b200 import synthetic as S
    tr = Transcriber("small_v2", "cuda", synthetic=True)
    w = S.make_waveforms(1, 320000, seed=21)[0]
    t = tr.transcribe(w, "eng")
    A, n = tr.engine.harvest_attention()
    st = tr.engine._last_search_state
    F = st["S_enc"] - 2
    assert 120 <= F <= 126
    stamps = tr.engine.token_timestamps(3)[0]
    if n[0]:
        assert stamps[0] == start_bins(A[0, :n[0], 1:1 + F].double().cpu().numpy(), 3)
        assert len(t.tokens) >= 1 and all(0.0 <= x.time_s <= 20.0 for x in t.tokens)
        assert all(0.0 < x.prob <= 1.0 for x in t.tokens)
    sums = A[0, :n[0]].sum(-1).cpu()
    assert torch.allclose(sums, torch.full_like(sums, 16.0), atol=1e-3)  # 16 heads, each a distribution over the frames
