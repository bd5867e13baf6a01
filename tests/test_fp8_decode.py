"""FP8 decoder weights (weight-only E4M3, DESIGN.md section 16).

The mode is defined by `dequantize_decoder_weights`: an FP8 model computes exactly the fp16 model on W' = q * s.  CPU
tests pin the quantizer (against torch's round-to-nearest-even e4m3fn conversion, on random, all-zero, subnormal-range,
clamp-boundary and maximum-magnitude rows), the exactness of W' in fp16, the error bound and the error paths, and the
C-ABI argument checks of the two e4m3 entries.  GPU tests hold sb_gemm_decode_e4m3 / sb_vocab_proj_e4m3 bit for bit to
the fp16 kernels on W' (and within a bound of float64), and whole translations with FP8 weights bit for bit to fp16
translations of the dequantized weights."""
import ctypes as C
import math

import pytest
import torch

from seamless_communication_b200 import config as CF, synthetic as S
from seamless_communication_b200.models.fp8_weights import (decoder_weight_names, dequantize_decoder_weights,
                                                            dequantize_rows, quantize_rows)
from seamless_communication_b200.ops import decode_splits

dev = "cuda"
gpu = pytest.mark.gpu
SB_EINVAL = -1  # include/seamless_b200.h
E4M3 = torch.float8_e4m3fn


def _rows():
    """Rows of every kind the quantizer meets: random at many magnitudes, all zero, tiny (scale clamped at 2^-15, values
    in e4m3's subnormal range or flushed), exactly 448 * 2^e (largest value of a scale), just above it (next scale), and
    the largest magnitude accepted, 448 * 2^7."""
    g = torch.Generator().manual_seed(0)
    rows = [torch.randn(256, generator=g) * 2.0 ** e for e in range(-24, 14, 3)]
    rows.append(torch.zeros(256))
    rows.append(torch.randn(256, generator=g) * 2.0 ** -30)
    rows.append(torch.linspace(-2.0 ** -20, 2.0 ** -20, 256))
    for e in (-15, -3, 0, 7):
        r = torch.randn(256, generator=g) * 2.0 ** e
        r[7] = 448 * 2.0 ** e
        rows.append(r)
        if e < 7:
            r = r.clone()
            r[7] = 448 * 2.0 ** e * (1 + 2 ** -20)
            rows.append(r)
    r = torch.randn(256, generator=g)
    r[3] = -448 * 2.0 ** 7
    rows.append(r)
    return torch.stack(rows)


# ------------------------------------------------------------------------------------------------ CPU
def test_quantizer_scale_and_rounding():
    w = _rows()
    q, s = quantize_rows(w)
    assert q.dtype == E4M3 and s.dtype == torch.float32 and q.shape == w.shape and s.shape == (w.shape[0],)
    amax = w.abs().amax(1).double()
    for i in range(w.shape[0]):
        e = math.log2(float(s[i]))
        assert e == int(e) and -15 <= e <= 7, (i, float(s[i]))
        if amax[i] == 0:
            assert s[i] == 1.0
            continue
        assert amax[i] <= 448 * float(s[i])  # never saturates
        if e > -15:
            assert amax[i] > 448 * float(s[i]) / 2, i  # the smallest such power of two
    # q is torch's round-to-nearest-even e4m3fn conversion of W / s (an exact division)
    ref = (w.double() / s.double()[:, None]).float().to(E4M3)
    assert torch.equal(q.view(torch.uint8), ref.view(torch.uint8))


def test_dequantized_weights_exact_in_fp16_and_bounded():
    w = _rows()
    q, s = quantize_rows(w)
    wp = dequantize_rows(q, s)
    assert wp.dtype == torch.float16
    exact = q.double() * s.double()[:, None]
    assert torch.equal(wp.double(), exact)
    assert torch.equal(wp.float(), q.float() * s[:, None])
    # relative error <= 2^-4 wherever W / s is in e4m3's normal range (>= 2^-6)
    normal = (w.double() / s.double()[:, None]).abs() >= 2.0 ** -6
    err = ((exact - w.double()).abs() / w.double().abs())[normal]
    assert normal.sum() > 1000 and err.max().item() <= 2.0 ** -4


@pytest.mark.parametrize("bad", ["nan", "inf", "range"])
def test_quantizer_rejects(bad):
    w = torch.randn(4, 64)
    w[2, 5] = {"nan": float("nan"), "inf": -float("inf"), "range": 448 * 2.0 ** 7 * 1.001}[bad]
    with pytest.raises(ValueError):
        quantize_rows(w)
    with pytest.raises(ValueError):
        quantize_rows(torch.zeros(64))


@pytest.mark.parametrize("arch", ["tiny_v2", "tiny_v1"])
def test_dequantize_decoder_weights_names(arch):
    cfg = CF.UNITY_ARCHS[arch]()
    sd = S.make_unity_state_dict(cfg, 0, dec_gain=4.0, with_t2u=True)
    names = decoder_weight_names(sd, cfg)
    per_layer = ["self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.output_proj",
                 "encoder_decoder_attn.q_proj", "encoder_decoder_attn.output_proj", "ffn.inner_proj", "ffn.output_proj"]
    want = [f"text_decoder.layers.{i}.{p}.weight" for i in range(cfg.dec_layers) for p in per_layer]
    want += [k for k in ("text_decoder_frontend.embed.weight", "final_proj.weight") if k in sd]
    if arch == "tiny_v1":
        want += [f"t2u_model.decoder.layers.{i}.{p}.weight" for i in range(cfg.t2u_dec_layers) for p in per_layer]
        want += [k for k in ("t2u_model.decoder_frontend.embed.weight", "t2u_model.final_proj.weight") if k in sd]
    assert names == want
    out = dequantize_decoder_weights(sd, cfg)
    assert set(out) == set(sd)
    for k in sd:
        if k in names:
            q, s = quantize_rows(sd[k])
            assert out[k].dtype == torch.float16 and torch.equal(out[k], dequantize_rows(q, s)), k
        else:  # K|V projections, biases, LayerNorms, the encoder and the NAR T2U are untouched
            assert out[k] is sd[k], k
    assert not any("encoder_decoder_attn.k_proj" in k or "encoder_decoder_attn.v_proj" in k or k.endswith(".bias")
                   for k in names)


def _desc(**kw):
    from seamless_communication_b200._lib import GemmDesc
    d = GemmDesc()
    d.a, d.a_rows, d.a_ld, d.c_in, d.taps, d.dil, d.a_row0 = 0x10000, 160, 1024, 1024, 1, 1, 0
    d.w, d.n, d.m = 0x20000, 1024, 160
    d.out, d.out_ld, d.out_f32, d.alpha, d.gamma = 0x40000, 1024, 1, 1.0, 1.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("case", ["scale_null", "scale_misaligned", "w_misaligned", "a_misaligned", "a_ld", "c_in", "taps",
                                  "glu", "res1", "masked", "splits0", "splits_big", "slice_rows", "direct_splits",
                                  "direct_f32", "direct_act", "partials_misaligned"])
def test_gemm_decode_e4m3_argument_checks(case):
    """sb_gemm_decode_e4m3 refuses before touching the device (fake addresses are never dereferenced)."""
    from seamless_communication_b200 import _lib
    lib = _lib.load()
    scale, splits, part, sr = 0x30000, 2, 0x50000, 256
    d = _desc(out=0, out_f32=0)
    if case == "scale_null": scale = 0
    elif case == "scale_misaligned": scale = 0x30002
    elif case == "w_misaligned": d.w = 0x20008
    elif case == "a_misaligned": d.a = 0x10008
    elif case == "a_ld": d.a_ld = 1020
    elif case == "c_in": d.c_in = 1000
    elif case == "taps": d.taps = 3
    elif case == "glu": d.glu = 1
    elif case == "res1": d.res1 = 0x60000
    elif case == "masked": d.seq_rows = 10
    elif case == "splits0": splits = 0
    elif case == "splits_big": splits = 17
    elif case == "slice_rows": sr = 100
    elif case.startswith("direct"):
        part, splits, d.out, d.out_f32, d.act = None, 1, 0x40000, 0, 1
        if case == "direct_splits": splits = 2
        elif case == "direct_f32": d.out_f32 = 1
        else: d.act = 2
    elif case == "partials_misaligned": part = 0x50004
    assert lib.sb_gemm_decode_e4m3(C.byref(d), scale, splits, part, sr, None) == SB_EINVAL
    assert b"e4m3" in lib.sb_last_error()


@pytest.mark.parametrize("case", ["scale_null", "scale_misaligned", "w_misaligned", "out_misaligned", "out_ld", "out_f16",
                                  "act", "prefetch", "c_in", "glu", "stats_misaligned", "out_ld_short"])
def test_vocab_proj_e4m3_argument_checks(case):
    from seamless_communication_b200 import _lib
    lib = _lib.load()
    scale = 0x30000
    d = _desc(n=1000, out_ld=1000)
    if case == "scale_null": scale = 0
    elif case == "scale_misaligned": scale = 0x30001
    elif case == "w_misaligned": d.w = 0x20004
    elif case == "out_misaligned": d.out = 0x40008
    elif case == "out_ld": d.out_ld = 1002
    elif case == "out_f16": d.out_f32 = 0
    elif case == "act": d.act = 1
    elif case == "prefetch": d.prefetch, d.prefetch_bytes = 0x70000, 4096
    elif case == "c_in": d.c_in = 96
    elif case == "glu": d.glu = 1
    elif case == "stats_misaligned": d.tile_stats = 0x80004
    elif case == "out_ld_short": d.out_ld = 996
    assert lib.sb_vocab_proj_e4m3(C.byref(d), scale, None) == SB_EINVAL
    assert b"e4m3" in lib.sb_last_error()


def test_load_unity_model_rejects_other_dtypes():
    from seamless_communication_b200.engine import UnitYEngine
    with pytest.raises(ValueError, match="decoder_weight_dtype"):
        UnitYEngine(CF.tiny_v2(), {}, (None, None), decoder_weight_dtype=torch.bfloat16)


# ------------------------------------------------------------------------------------------------ GPU: kernels
M, FFN = 1024, 8192


def _weights(n, k, seed, spread=True):
    """Rows whose scales cover the whole clamp range [2^-15, 2^7] (spread: row magnitudes from 448 * 2^-16 to 448 * 2^7),
    or ~N(0, 1/k) rows; fp16 W' and (q, s)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(n, k, generator=g) / math.sqrt(k)
    if spread:
        w = w * torch.pow(2.0, torch.randint(-3, 18, (n, 1), generator=g).float())
        w[1::97] = 0.0
    q, s = quantize_rows(w)
    return dequantize_rows(q, s).to(dev), q.to(dev), s.to(dev)


def _act(rows, k, seed):
    from seamless_communication_b200.ops import Seq
    g = torch.Generator().manual_seed(seed)
    return Seq(1, rows, k, buf=torch.randn(rows, k, generator=g).half().to(dev))


def _chunks(rows):
    return [(r0, min(rows, r0 + 256)) for r0 in range(0, rows, 256)]


@gpu
@pytest.mark.parametrize("rows", [1, 5, 35, 160, 256, 320])
@pytest.mark.parametrize("n,k", [(3 * M, M), (M, M), (M, FFN)], ids=["qkv", "attn", "ffn_out"])
def test_splitk_e4m3_equals_fp16_on_dequantized(rows, n, k):
    """Split-K partials at the step's K slices for this row count and at one slice: bit-identical to sb_gemm_decode on
    W' (per chunk of 256 rows past 256), with scales across the clamp range; within 1e-3 of float64 on normal rows."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.ops import Seq
    wp, q, s = _weights(n, k, n + k)
    a = _act(rows, k, rows)
    qkv, attn, ffn = decode_splits(rows, M, FFN)
    SR = ops.slice_rows(rows)
    for splits in sorted({{(3 * M, M): qkv, (M, M): attn, (M, FFN): ffn}[(n, k)], 1}):
        got = torch.full((splits * SR, n), float("nan"), device=dev)
        ops.gemm_splitk_e4m3(a, q, s, n, splits, got)
        want = torch.full_like(got, float("nan"))
        for r0, r1 in _chunks(rows):
            sub = Seq(1, r1 - r0, k, buf=a.buf[r0:r1])
            part = torch.full(((splits) * ops.slice_rows(r1 - r0), n), float("nan"), device=dev)
            ops.gemm_splitk(sub, wp, n, splits, part, transposed=True)
            want.view(splits, SR, n)[:, r0:r1] = part.view(splits, -1, n)[:, :r1 - r0]
        g3, w3 = got.view(splits, SR, n)[:, :rows], want.view(splits, SR, n)[:, :rows]
        assert torch.equal(g3, w3), (splits, (g3 - w3).abs().max().item())
    wn, qn, sn = _weights(n, k, n + k + 1, spread=False)
    part = torch.empty((SR, n), device=dev)
    ops.gemm_splitk_e4m3(a, qn, sn, n, 1, part)
    ref = a.buf.double() @ wn.double().t()
    assert (part[:rows].double() - ref).abs().max().item() < 1e-3


@gpu
@pytest.mark.parametrize("rows", [1, 5, 35, 160, 256, 320])
def test_ffn_inner_e4m3_equals_fp16_on_dequantized(rows):
    """Direct mode (fp16 relu(a . W'^T + bias)), bit for bit against sb_gemm_decode on W', per chunk past 256 rows."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.ops import ACT_RELU, Seq
    wp, q, s = _weights(FFN, M, 3)
    bias = torch.randn(FFN, device=dev)
    a = _act(rows, M, rows + 1)
    got = ops.gemm_decode_e4m3(a, q, s, FFN, bias, act=ACT_RELU)
    want = torch.empty_like(got.buf)
    for r0, r1 in _chunks(rows):
        want[r0:r1] = ops.gemm_decode(Seq(1, r1 - r0, M, buf=a.buf[r0:r1]), wp, FFN, bias, act=ACT_RELU).buf
    assert torch.equal(got.buf, want)


@gpu
@pytest.mark.parametrize("rows", [5, 160, 320])
@pytest.mark.parametrize("V", [129, 1126, 1663, 1664, 1665, 8294])
def test_vocab_proj_e4m3_equals_fp16_on_dequantized(rows, V):
    """Logits and tile statistics bit-identical to the fp16 projection on W' (sb_gemm with tile_stats, per chunk of 256
    rows) at V on both sides of one tile and of K+2 = 13 tiles; the tile top-K on them gives the same candidates; the
    logits are within 1e-3 of float64."""
    from seamless_communication_b200 import _lib, ops
    from seamless_communication_b200.ops import Seq
    K = 11
    wp, q, s = _weights(V, M, V, spread=False)
    s_spread = s * torch.pow(2.0, torch.randint(-3, 4, (V,), device=dev).float())  # scales vary across features too
    q_wp = dequantize_rows(q.cpu(), s_spread.cpu()).to(dev)
    a = _act(rows, M, V + rows)
    ld = (V + 7) // 8 * 8
    T = (V + 127) // 128
    for scale, w16 in ((s, wp), (s_spread, q_wp)):
        out = Seq(1, rows, V, dtype=torch.float32, buf=torch.full((rows, ld), float("nan"), device=dev))
        stats = torch.full((T, rows, 2), float("nan"), device=dev)
        ops.vocab_proj_e4m3(a, q, scale, V, out, stats)
        want = torch.full((rows, ld), float("nan"), device=dev)
        wstats = torch.full((T, rows, 2), float("nan"), device=dev)
        for r0, r1 in _chunks(rows):
            o = Seq(1, r1 - r0, V, dtype=torch.float32, buf=torch.empty((r1 - r0, ld), device=dev))
            st = torch.empty((T, r1 - r0, 2), device=dev)
            ops.gemm(Seq(1, r1 - r0, M, buf=a.buf[r0:r1]), w16, V, None, out=o, out_f32=True, tile_stats=st)
            want[r0:r1, :V] = o.buf[:, :V]
            wstats[:, r0:r1] = st
        assert torch.equal(out.buf[:, :V], want[:, :V])
        assert torch.equal(stats, wstats)
        lib = _lib.load()
        cands = []
        for lg, stt in ((out.buf, stats), (want, wstats)):
            cv = torch.empty((rows, K), device=dev)
            ci = torch.empty((rows, K), dtype=torch.int32, device=dev)
            el = torch.empty((rows,), device=dev)
            _lib.check(lib.sb_logits_topk_tiles(lg.data_ptr(), ld, stt.data_ptr(), rows, V, 0, 2, 3, 0.0, K, cv.data_ptr(),
                                                ci.data_ptr(), el.data_ptr(), ops._stream()), "sb_logits_topk_tiles")
            cands.append((cv, ci, el))
        assert all(torch.equal(x, y) for x, y in zip(*cands))
    ref = a.buf.double() @ wp.double().t()
    o = Seq(1, rows, V, dtype=torch.float32, buf=torch.empty((rows, ld), device=dev))
    ops.vocab_proj_e4m3(a, q, s, V, o)
    assert (o.buf[:, :V].double() - ref).abs().max().item() < 1e-3


# ------------------------------------------------------------------------------------------------ GPU: end to end
def _pair(arch, seed=0):
    """(FP8 model, fp16 model of the dequantized weights, vocoder) of one architecture's synthetic weights."""
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    cfg = CF.UNITY_ARCHS[arch]()
    sd = S.make_unity_state_dict(cfg, seed, dec_gain=4.0, with_t2u=True)
    toks = S.make_tokenizers(cfg)
    f8 = load_unity_model(arch, state_dict=sd, tokenizers=toks, decoder_weight_dtype=torch.float8_e4m3fn)
    f16 = load_unity_model(arch, state_dict=dequantize_decoder_weights(sd, cfg), tokenizers=toks)
    vc = CF.tiny_vocoder()
    voc = load_vocoder_model("tiny", state_dict=S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True))
    return cfg, sd, toks, f8, f16, voc


def _same(a, b):
    (t0, s0), (t1, s1) = a, b
    assert t0 == t1
    if s0 is None:
        assert s1 is None
        return
    assert s0.units == s1.units
    assert len(s0.audio_wavs) == len(s1.audio_wavs) and all(torch.equal(x, y) for x, y in zip(s0.audio_wavs, s1.audio_wavs))


def _translations(model, voc, v1, tasks=("s2tt", "s2st")):
    from seamless_communication_b200.inference import NGramRepeatBlockProcessor, SequenceGeneratorOptions, Translator
    tr = Translator(model, voc, device="cuda:0")
    src = tr.fbank_batch(S.make_waveforms(3, 32000, seed=11), torch.tensor([32000, 17000, 25000]))
    opts = SequenceGeneratorOptions(hard_max_seq_len=20)
    ngram = SequenceGeneratorOptions(hard_max_seq_len=20, step_processor=NGramRepeatBlockProcessor(2))
    kw = dict(unit_generation_opts=SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40)) if v1 else {}
    out = []
    for task in tasks:
        out.append(tr.predict(src, task, "spa", text_generation_opts=opts, **kw))
        out.append(tr.predict(src, task, "spa", text_generation_opts=ngram, **kw))
    return out


@gpu
@pytest.mark.parametrize("arch", ["tiny_v2", "small_v2", "tiny_v1", "small_v1"])
def test_translator_fp8_equals_fp16_on_dequantized(arch):
    """Translator(decoder_weight_dtype=float8_e4m3fn): texts, units and waveforms of S2TT and S2ST (S2TT only on the
    small archs) on a ragged batch, with and without n-gram blocking, equal an fp16 Translator of
    dequantize_decoder_weights(sd) bit for bit (tiny_v1: the AR unit search runs on e4m3 weights too).  The FP8 engines hold e4m3 weights; the fp16 ones do not."""
    cfg, sd, toks, f8, f16, voc = _pair(arch)
    v1 = cfg.encoder_variant == "v1"
    assert f8.engine.fp8 and not f16.engine.fp8 and "text_embed.q8" in f8.engine.w and "text_embed.q8" not in f16.engine.w
    if v1:
        assert f8.t2u_model.unit_engine.fp8 and f8.t2u_model.unit_engine.w["text_embed.q8"].dtype == E4M3
    # the tiny vocoder's 256-entry unit table only fits the tiny archs' units: the small archs run S2TT
    tasks = ("s2tt", "s2st") if arch.startswith("tiny") else ("s2tt",)
    a, b = _translations(f8, voc, v1, tasks), _translations(f16, voc, v1, tasks)
    for x, y in zip(a, b):
        _same(x, y)
    # the fp16 copies the FP8 engine keeps are the dequantized weights
    for k in ("text_embed", "text_decoder.layers.0.self_attn.qkv.w", "text_decoder.layers.0.ffn.inner_proj.w"):
        assert torch.equal(f8.engine.w[k], f16.engine.w[k]), k


@gpu
def test_banned_sequences_fp8_equals_fp16():
    """The search with banned sequences (MinTox's re-decode path) on e4m3 weights equals the fp16 search on W'."""
    from seamless_communication_b200.ops import Seq
    cfg, sd, toks, f8, f16, voc = _pair("tiny_v2", seed=3)
    g = torch.Generator().manual_seed(5)
    B, T = 4, 30
    enc = torch.randn(B * T, cfg.model_dim, generator=g).half().to(dev)
    lens = torch.tensor([30, 21, 30, 9], dtype=torch.int32, device=dev)
    prefix = [cfg.text_eos, 7]
    ban = [[11, 12], [40], [5, 6, 7]]
    res = []
    for m in (f8, f16):
        e = Seq(B, T, cfg.model_dim, buf=enc.clone())
        res.append(m.engine.beam_search(e, lens, prefix, beam=5, hard_max=25, banned=ban))
    assert res[0] == res[1]


@gpu
def test_fp8_hypotheses_match_oracle_on_dequantized():
    """The FP8 text search on tiny_v2 against the fp32 CPU oracle run on W': identical hypotheses, or a near-tie of the
    oracle's own scores (the existing audit of smoke())."""
    from oracle.unity_oracle import UnityOracle, s2st
    from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator
    cfg, sd, toks, f8, f16, voc = _pair("tiny_v2")
    waves = S.make_waveforms(2, 32000)
    tr = Translator(f8, voc, device="cuda:0")
    tr.predict(tr.fbank_batch(waves), "s2tt", "spa",
               text_generation_opts=SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=20))
    hyps = Translator._last_generator.last_text_output.hypotheses
    from oracle.unity_oracle import VocoderOracle
    wsd = {k: v.float() for k, v in dequantize_decoder_weights(sd, cfg).items()}  # the fp32 oracle: W' is exact in fp32
    uo = UnityOracle(cfg.to_dict(), wsd, toks)
    vc = CF.tiny_vocoder()
    ref = s2st(uo, VocoderOracle(vc.to_dict(), S.make_vocoder_state_dict(vc, 1)), waves, "spa", 25, 45, hard_max=20)
    for i in range(2):
        if hyps[i][0][1] != ref["text_ids"][i]:
            ids = torch.tensor(hyps[i][0][1])[None]
            h = uo.decoder(uo.embed_text(ids[:, :-1], 0), ref["enc"][i:i + 1], None)
            lp = torch.log_softmax(uo.project(h).float(), -1)[0]
            sc = sum(float(lp[t, ids[0, t + 1]]) for t in range(ids.shape[1] - 1)) / (ids.shape[1] - 1)
            assert abs(sc - ref["hyps"][i][0][0]) < 2e-2, i


@gpu
def test_two_lanes_equal_serial_fp8():
    """Two LanePool lanes over an FP8 tiny_v1 model (both engines) give the serial results bit for bit."""
    from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator
    from seamless_communication_b200.parallel import LanePool
    cfg, sd, toks, f8, f16, voc = _pair("tiny_v1", seed=2)
    tr = Translator(f8, voc, device="cuda:0")

    def run(w):
        return tr.predict(tr.fbank_batch(w), "s2st", "spa", text_generation_opts=SequenceGeneratorOptions(hard_max_seq_len=20),
                          unit_generation_opts=SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40))
    batches = [S.make_waveforms(2, 24000, seed=s) for s in (5, 6, 7)]
    serial = [run(w) for w in batches]
    pool = LanePool("cuda", 2, f8.engines)
    try:
        par = pool.map(run, [[w] for w in batches])
    finally:
        pool.close()
    for x, y in zip(serial, par):
        _same(x, y)
