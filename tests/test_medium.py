"""seamlessM4T_medium: the third SeamlessM4T card, on the v1 encoder, decoder-step and unit-search kernels.

CPU tests pin the `medium` architecture and the NLLB-200 language list to what the reference states
(tests/golden/medium_card.json, made by make_golden_medium.py), the synthetic NLLB-200 tokenizer layout, the loader's
architecture check and the fairseq checkpoint conversion at medium's layer counts and vocabulary.  GPU tests run at
medium's full width on synthetic weights: the decoder-step GEMMs at its FFN shapes and the vocabulary projection and
top-K at V = 256 206 against float64, and `Translator.predict` (S2ST, S2TT, ASR) on ragged batches against the fp32
oracle on the same padded batches, with FP8
weights, two lanes and a fairseq-named checkpoint."""
import dataclasses
import json
import math
import os
import types

import pytest
import torch

from seamless_communication_b200 import config as C, synthetic as S
from seamless_communication_b200.models import checkpoint as ck
from seamless_communication_b200.models.unity.model import check_state_dict

G = os.path.join(os.path.dirname(__file__), "golden")
dev = "cuda"
gpu = pytest.mark.gpu
V_MED = 256206


def golden():
    return json.load(open(os.path.join(G, "medium_card.json")))


def tiny_medium():
    """medium's layer counts and vocabulary at test widths: every parameter name and count of the real model."""
    return dataclasses.replace(C.medium(), name="tiny_medium", model_dim=128, num_heads=2, enc_ffn_dim=256,
                               dec_ffn_dim=256, t2u_ffn_dim=256)


# ------------------------------------------------------------------------------------------------ CPU
def test_medium_config_matches_reference():
    """`medium` against `_medium` / `_medium_t2u` (read with ast) and the seamlessM4T_medium card; every field the
    reference does not set for medium is base's, `max_seq_len` included."""
    d = golden()
    b, t, card = d["builder"]["medium"], d["t2u_builder"]["medium"], d["cards"]["seamlessM4T_medium"]
    m = C.medium()
    assert C.MODEL_CARDS[card["name"]] == card["model_arch"] == m.name == "medium"
    assert C.UNITY_ARCHS["medium"]().to_dict() == m.to_dict()
    assert b["archs"] == {"w2vbert_archs": "300m", "nllb_archs": "dense_600m", "unity_t2u_archs": "medium"}
    # recalled (fairseq2 is not in the reference tree): "300m" = 12 Conformer layers, "dense_600m" = 12 layers, FFN 4096
    assert (m.encoder_variant, m.enc_layers, m.dec_layers, m.dec_ffn_dim) == ("v1", 12, 12, 4096)
    assert m.text_vocab == b["text_vocab"] == V_MED
    # the adaptor is base's: one layer, kernel 8, stride 8, no GELU, no Conformer adaptor
    assert b["config"] == d["builder"]["base"]["config"]
    assert (b["config"]["num_adaptor_layers"], m.adaptor_kernel, m.adaptor_stride, m.model_dim) == \
           (1, b["config"]["adaptor_kernel_size"], b["config"]["adaptor_stride"], b["config"]["model_dim"])
    assert (m.t2u_enc_layers, m.t2u_dec_layers, m.t2u_ffn_dim, m.unit_max_seq_len) == \
           (t["num_encoder_layers"], t["num_decoder_layers"], t["ffn_inner_dim"], t["unit_max_seq_len"]) == (4, 4, 8192, 2048)
    assert m.num_heads == t["num_encoder_attn_heads"] == t["num_decoder_attn_heads"] and m.model_dim == t["model_dim"]
    vi = t["target_vocab_info"]
    assert (m.unit_vocab, m.unit_unk, m.unit_bos, m.unit_eos, m.unit_pad) == \
           (vi["size"], vi["unk_idx"], vi["bos_idx"], vi["eos_idx"], vi["pad_idx"])
    assert m.num_units == card["num_units"] and list(m.unit_langs) == card["unit_langs"] == \
           d["cards"]["seamlessM4T_large"]["unit_langs"]
    assert card["base"] == "unity_nllb-200" and list(m.langs) == list(C.NLLB200_LANGS) == d["cards"]["unity_nllb-200"]["langs"]
    assert len(C.NLLB200_LANGS) == 202
    # everything else is seamlessM4T_large's
    same = dataclasses.replace(m, name="base", enc_layers=24, dec_layers=24, dec_ffn_dim=8192, text_vocab=256102,
                               t2u_enc_layers=6, t2u_dec_layers=6, langs=C.NLLB100_LANGS)
    assert same == C.base()
    assert C.base().max_seq_len == m.max_seq_len == 4096
    # vocoder_36langs serves medium (docs/m4t/README.md)
    assert d["readme_vocoder_lines"] and "seamlessM4T_medium" in d["readme_vocoder_lines"][0]
    assert C.VOCODER_CARDS["vocoder_36langs"] == "base"


def test_nllb200_tokenizer_layout_and_prefixes():
    """The synthetic tokenizer of medium: 256 206 pieces, the 202 `__lang__` symbols in card order, the 3 data-source
    symbols last; the target prefix [</s>, __lang__] of the first, last and some other languages."""
    tok, _ = S.make_tokenizers(C.medium())
    assert tok.vocab_info.size == len(tok.model.pieces) == V_MED
    n = len(C.NLLB200_LANGS)
    first = V_MED - 3 - n
    assert [tok.model.index_to_token(first + i) for i in range(n)] == [f"__{lang}__" for lang in C.NLLB200_LANGS]
    assert [tok.model.index_to_token(V_MED - 3 + i) for i in range(3)] == ["<MINED_DATA>", "<MMT_BT_DATA>", "<SMT_BT_DATA>"]
    want = {"ace": first, "ace_Latn": first + 1, "eng": first + 46, "spa": first + C.NLLB200_LANGS.index("spa"),
            "cmn_Hant": V_MED - 5, "zul": V_MED - 4}
    assert want["eng"] == first + C.NLLB200_LANGS.index("eng")
    for lang, idx in want.items():
        assert tok.lang_index(lang) == idx
        enc = tok.create_encoder(task="translation", lang=lang, mode="target")
        assert enc.prefix_indices.tolist() == [C.medium().text_eos, idx], lang
    # seamlessM4T_large's tokenizer is unchanged: NLLB-100 layout
    tl, _ = S.make_tokenizers(C.base())
    assert tl.vocab_info.size == 256102 and tl.lang_index("zul") == 256102 - 4


def test_architecture_check():
    """check_state_dict on a tiny copy with medium's names: each kind of mismatch raises ValueError naming it, the right
    state dict passes, and load_unity_model("seamlessM4T_medium") refuses large's layer counts before building
    anything."""
    cfg = tiny_medium()
    sd = S.make_unity_state_dict(cfg, 0, with_t2u=True)
    check_state_dict(sd, cfg)
    check_state_dict({k: v for k, v in sd.items() if not k.startswith("t2u_model.")}, cfg)  # S2TT-only weights

    def drop(prefix):
        return {k: v for k, v in sd.items() if not k.startswith(prefix)}
    cases = [("speech encoder layers 11", drop("speech_encoder.inner.layers.11.")),
             ("text decoder layers 11", drop("text_decoder.layers.11.")),
             ("T2U encoder layers 3", drop("t2u_model.encoder.layers.3.")),
             ("T2U decoder layers 3", drop("t2u_model.decoder.layers.3."))]
    ffn = dict(sd)
    ffn["text_decoder.layers.0.ffn.inner_proj.weight"] = torch.zeros(2 * cfg.dec_ffn_dim, cfg.model_dim)
    cases.append(("text decoder FFN width 512", ffn))
    voc = dict(sd)
    voc["final_proj.weight"] = voc["text_decoder_frontend.embed.weight"] = torch.zeros(256102, cfg.model_dim)
    cases.append(("text vocabulary size 256102", voc))
    more = dict(sd)
    more["text_decoder.layers.12.ffn.inner_proj.weight"] = sd["text_decoder.layers.0.ffn.inner_proj.weight"]
    cases.append(("text decoder layers 13", more))
    for what, bad in cases:
        with pytest.raises(ValueError, match=what):
            check_state_dict(bad, cfg)
    from seamless_communication_b200.models.unity import load_unity_model
    big = S.make_unity_state_dict(dataclasses.replace(cfg, enc_layers=24, dec_layers=24), 0)
    with pytest.raises(ValueError, match="'medium': speech encoder layers 24, the architecture has 12"):
        load_unity_model("seamlessM4T_medium", device="cpu", state_dict=big, tokenizers=S.make_tokenizers(cfg))


def fairseq_medium_checkpoint(sd):
    """The fairseq-named multitask checkpoint of a medium-named state dict with its AR T2U: speech encoder and text
    decoder under fairseq names (test_v1_encoder.to_fairseq), T2U under synthesizer_encoder / decoder, the tied table in
    fairseq's (BOS, PAD, EOS, UNK) order, and a text encoder that loading drops."""
    from test_v1_s2st import fairseq_ar_checkpoint
    out = fairseq_ar_checkpoint(sd)
    out["model"]["text_encoder.layers.0.fc1.weight"] = torch.zeros(4, 4)
    return out


def test_fairseq_medium_checkpoint_converts():
    """At medium's layer counts and vocabulary: every fairseq key converts to exactly one fairseq2 key, the result is
    the state dict the checkpoint was made from (tied table unified and its control rows permuted back, as for large),
    the text decoder's embedding and projection are one tensor, and a dummy 256 207th row is discarded."""
    cfg = tiny_medium()
    sd = S.make_unity_state_dict(cfg, 0, with_t2u=True)
    fs = fairseq_medium_checkpoint(sd)
    names = [ck.rename_key(k) for k in fs["model"]]
    assert len(set(names)) == len(names)
    out = ck.convert_unity_checkpoint(fs, nllb_vocab=cfg.text_vocab)["model"]
    assert sorted(out) == sorted(list(sd) + ["text_encoder.layers.0.ffn.inner_proj.weight", "text_encoder_frontend.embed.weight"])
    for k in sd:
        assert torch.equal(out[k], sd[k]), k
    assert out["final_proj.weight"] is out["text_decoder_frontend.embed.weight"]
    assert out["t2u_model.decoder_frontend.embed.weight"] is out["t2u_model.final_proj.weight"]
    assert out["final_proj.weight"].shape == (V_MED, cfg.model_dim)
    check_state_dict(out, cfg)
    fs = fairseq_medium_checkpoint(sd)
    emb = fs["model"]["target_letter_decoder.output_projection.weight"]
    fs["model"]["target_letter_decoder.output_projection.weight"] = torch.cat([emb, torch.ones(1, cfg.model_dim)])
    out = ck.convert_unity_checkpoint(fs, nllb_vocab=cfg.text_vocab)["model"]
    assert torch.equal(out["final_proj.weight"], sd["final_proj.weight"])


def test_text_input_on_medium_raises():
    """T2ST and T2TT raise on medium as on large: text input needs the NLLB text encoder."""
    from seamless_communication_b200.inference import Translator
    tr = Translator.__new__(Translator)
    tr.model, tr.apply_mintox = types.SimpleNamespace(config=C.medium(), t2u_model=object()), False
    for task in ("t2st", "t2tt"):
        with pytest.raises(NotImplementedError, match="text"):
            tr.predict(torch.zeros(4), task, "spa", src_lang="eng")


def test_medium_step_shapes():
    """The decoder-step shapes of medium the GPU tests below cover: FFN out at (2, 8, 8) K slices for 160 rows, 2002
    projection tiles of which the last is 78 wide, a row stride of 256 208."""
    from seamless_communication_b200.ops import decode_splits
    assert decode_splits(160, 1024, 4096) == (2, 8, 8)
    assert (V_MED + 127) // 128 == 2002 and V_MED - 2001 * 128 == 78 and V_MED % 8 == 6


# ------------------------------------------------------------------------------------------------ GPU: kernels
M, FFN, ROWS = 1024, 4096, 160


def _act(rows, k, seed):
    from seamless_communication_b200.ops import Seq
    g = torch.Generator().manual_seed(seed)
    return Seq(1, rows, k, buf=torch.randn(rows, k, generator=g).half().to(dev))


def _weight16(n, k, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, k, generator=g) / math.sqrt(k)).half()


@gpu
def test_ffn_inner_and_out_at_medium_shapes_match_float64():
    """sb_gemm_decode at medium's FFN shapes and 160 rows: FFN inner (1024 -> 4096, bias + ReLU, direct mode: 32 CTAs)
    and FFN out (4096 -> 1024 at the step's 8 K slices), fp16 and e4m3 weights, against float64; the e4m3 entries bit
    for bit against fp16 on W' = q * s.  Output columns past 4096 and slices past 8 keep their NaN."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.models.fp8_weights import dequantize_rows, quantize_rows
    from seamless_communication_b200.ops import ACT_RELU, Seq
    splits = ops.decode_splits(ROWS, M, FFN)[2]
    assert splits == 8
    g = torch.Generator().manual_seed(3)
    bias = torch.randn(FFN, generator=g).to(dev)
    a = _act(ROWS, M, 1)
    w = _weight16(FFN, M, 2)
    q, s = quantize_rows(w.float())
    wp = dequantize_rows(q, s)
    for name, w16 in (("fp16", w.to(dev)), ("e4m3", wp.to(dev))):
        big = torch.full((ROWS, FFN + 8), float("nan"), device=dev).half()
        out = Seq(1, ROWS, FFN, buf=big[:, :FFN])
        if name == "fp16":
            ops.gemm_decode(a, w16, FFN, bias, act=ACT_RELU, out=out)
        else:
            ops.gemm_decode_e4m3(a, q.to(dev), s.to(dev), FFN, bias, act=ACT_RELU, out=out)
            want = ops.gemm_decode(a, w16, FFN, bias, act=ACT_RELU)
            assert torch.equal(big[:, :FFN], want.buf)
        ref = torch.relu(a.buf.double() @ w16.double().t() + bias.double())
        got = big[:, :FFN].double()
        assert ((got - ref).abs() <= 2e-3 + 1e-3 * ref.abs()).all(), (name, (got - ref).abs().max().item())
        assert torch.isnan(big[:, FFN:]).all(), name
    # FFN out: K = 4096 in 8 slices of 8 k-blocks
    a = _act(ROWS, FFN, 4)
    w = _weight16(M, FFN, 5)
    q, s = quantize_rows(w.float())
    wp = dequantize_rows(q, s).to(dev)
    SR = ops.slice_rows(ROWS)
    for name, w16 in (("fp16", w.to(dev)), ("e4m3", wp)):
        part = torch.full(((splits + 1) * SR, M), float("nan"), device=dev)
        if name == "fp16":
            ops.gemm_splitk(a, w16, M, splits, part, transposed=True)
        else:
            ops.gemm_splitk_e4m3(a, q.to(dev), s.to(dev), M, splits, part)
            want = torch.full_like(part, float("nan"))
            ops.gemm_splitk(a, w16, M, splits, want, transposed=True)
            assert torch.equal(part.view(splits + 1, SR, M)[:splits, :ROWS], want.view(splits + 1, SR, M)[:splits, :ROWS])
        p = part.view(splits + 1, SR, M)
        assert torch.isnan(p[splits]).all() and torch.isnan(p[:splits, ROWS:]).all(), name
        err = (p[:splits, :ROWS].double().sum(0) - a.buf.double() @ w16.double().t()).abs().max().item()
        assert err < 1e-3, (name, err)


@gpu
def test_vocab_projection_and_topk_at_v256206():
    """The tied projection with tile statistics at V = 256 206 (2002 tiles, the last 78 wide; 256 206 % 8 = 6) on fp16
    and e4m3 weights at 160 rows: logits within 1e-3 of float64, the statistics those of the stored logits (the
    padding does not enter them), e4m3 bit for bit the fp16 projection on W'.  The two columns of row-stride padding past
    256 206 start as NaN sentinels; the row's last 8-column store may write 0 there, and nothing else is written.
    sb_logits_topk_tiles and sb_logits_topk_tiles_ban on those logits and statistics give the float64 top-K, with the
    padding holding NaN and then values that would win if read; so does the two-pass path on adversarial rows."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.models.fp8_weights import dequantize_rows, quantize_rows
    from seamless_communication_b200.ops import Seq
    from test_search_select import EOS, PAD, PEN, UNK, _assert_matches, _device_rows, _rows
    from test_mintox import _topk
    V, K, R = V_MED, 11, ROWS
    ld = (V + 7) // 8 * 8
    T = (V + 127) // 128
    assert ld - V == 2 and T == 2002
    g = torch.Generator().manual_seed(206)
    w = (torch.randn(V, M, generator=g) * 0.05).half()
    q, s = quantize_rows(w.float())
    wp = dequantize_rows(q, s)
    a = _act(R, M, 7)
    res = {}
    for name, w16 in (("fp16", w), ("fp16 on W'", wp), ("e4m3", wp)):
        w16 = w16.to(dev)
        out = Seq(1, R, V, dtype=torch.float32, buf=torch.full((R, ld), float("nan"), device=dev))
        stats = torch.full((T, R, 2), float("nan"), device=dev)
        if name != "e4m3":
            ops.gemm(a, w16, V, None, out=out, out_f32=True, tile_stats=stats)
        else:
            ops.vocab_proj_e4m3(a, q.to(dev), s.to(dev), V, out, stats)
        torch.cuda.synchronize()
        lg = out.buf
        assert torch.isfinite(lg[:, :V]).all(), name
        # the last 8-column store of a row covers the two padding columns: they hold 0 or keep their NaN, nothing else
        pad = lg[:, V:]
        assert (torch.isnan(pad) | (pad == 0)).all(), name
        ref = a.buf.double() @ w16.double().t()
        assert (lg[:, :V].double() - ref).abs().max().item() < 1e-3, name
        tiles = lg.new_full((R, T * 128), -math.inf)
        tiles[:, :V] = lg[:, :V]
        tiles = tiles.view(R, T, 128)
        assert torch.equal(stats[:, :, 0].t(), tiles.max(-1).values), name
        assert torch.allclose(stats[:, :, 1].t(), torch.exp(tiles - tiles.max(-1, keepdim=True).values).sum(-1), rtol=1e-5)
        assert int((stats[-1, :, 1] <= 78).all()) and float(stats[-1, :, 1].min()) >= 1.0
        res[name] = (lg.clone(), stats.clone())
    assert torch.equal(res["fp16 on W'"][0][:, :V], res["e4m3"][0][:, :V]) and torch.equal(res["fp16 on W'"][1], res["e4m3"][1])
    lg, stats = res["fp16"]
    x = lg[:, :V].cpu()
    rows = list(range(0, R, 16)) + [R - 1]  # float64 top-K on 11 of the 160 rows, the kernels on all of them
    last = list(range(2001 * 128, V))
    bans = [[EOS] if r % 3 == 0 else ([int(x[r].argmax())] if r % 3 == 1 else last) for r in range(R)]
    for bait in (float("nan"), 1.0e4):
        lg[:, V:] = bait
        for b in (None, bans):
            cv, ci, el = _topk(lg, V, K, PAD, EOS, UNK, PEN, bans=b, tiles=True, stats=stats)
            sub = [bans[r] for r in rows] if b else None
            _assert_matches(cv[rows], ci[rows], el[rows], x[rows], K, sub, f"bait={bait} bans={b is not None}")
            assert int(ci.max()) < V
    # adversarial rows (PAD / UNK / EOS on top, ties across a tile boundary, one spike per tile, -inf entries) on both
    # paths, with the padding as NaN and as bait
    xa, abans = _rows(V, 2062)
    for bait in (float("nan"), 1.0e4):
        lga = _device_rows(xa, ld, bait)
        for tiles in (False, True):
            for b in (None, abans):
                cv, ci, el = _topk(lga, V, K, PAD, EOS, UNK, PEN, bans=b, tiles=tiles)
                _assert_matches(cv, ci, el, xa, K, b, f"bait={bait} tiles={tiles} bans={b is not None}")


# ------------------------------------------------------------------------------------------------ GPU: end to end
def _text_opts(**kw):
    from seamless_communication_b200.inference import SequenceGeneratorOptions
    return SequenceGeneratorOptions(hard_max_seq_len=20, **kw)


def _unit_opts(**kw):
    from seamless_communication_b200.inference import SequenceGeneratorOptions
    return SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40, **kw)


@pytest.fixture(scope="module")
def medium():
    """Full-width seamlessM4T_medium on seeded synthetic weights (the AR T2U's EOS reachable, as in test_v1_s2st), the
    vocoder_36langs architecture with a duration predictor, and the fp32 oracles on the same state dicts."""
    from oracle_v1 import UnityOracleV1
    from test_v1_s2st import unit_oracle, with_reachable_eos
    from seamless_communication_b200.inference import Translator
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    cfg, vc = C.medium(), C.base_vocoder()
    # an EOS row of 4.5 times the other rows' spread (seed 14): on the S2ST batch below the oracle's unit searches end
    # after 11 units on EOS and at the 40-unit budget
    sd = with_reachable_eos(S.make_unity_state_dict(cfg, 0, dec_gain=4.0, with_t2u=True), cfg, scale=4.5, seed=14)
    toks = S.make_tokenizers(cfg)
    vsd = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
    model = load_unity_model("seamlessM4T_medium", state_dict=sd, tokenizers=toks)
    voc = load_vocoder_model("vocoder_36langs", state_dict=vsd)
    return dict(cfg=cfg, sd=sd, toks=toks, vc=vc, vsd=vsd, model=model, voc=voc, tr=Translator(model, voc, device="cuda:0"),
                uo=UnityOracleV1(cfg.to_dict(), sd, toks), ou=unit_oracle(cfg, sd))


@gpu
def test_translator_builds_from_card():
    """Translator("seamlessM4T_medium", "vocoder_36langs", synthetic=True) resolves the card to `medium`, builds the
    AR T2U's unit engine at 4 layers and the vocoder with vocoder_36langs' speakers, and translates."""
    from seamless_communication_b200.inference import Translator
    from seamless_communication_b200.models.unity import UnitYT2UModel
    tr = Translator("seamlessM4T_medium", "vocoder_36langs", "cuda", synthetic=True)
    m = tr.model
    assert m.config.name == "medium" and m.config.text_vocab == V_MED and m.engine.cfg.dec_layers == 12
    assert isinstance(m.t2u_model, UnitYT2UModel) and len(m.engines) == 2
    ucfg = m.t2u_model.unit_engine.cfg
    assert (ucfg.dec_layers, ucfg.dec_ffn_dim, ucfg.text_vocab) == (4, 8192, 10082)
    assert tr.text_tokenizer.vocab_info.size == V_MED and tr.unit_tokenizer.vocab_info.size == 10082
    assert tr.vocoder.lang_spkr_idx_map == C.vocoder_lang_spkr_idx_map("vocoder_36langs")
    texts, speech = tr.predict(S.make_waveforms(1, 16000, seed=3)[0], "s2st", "spa", text_generation_opts=_text_opts(),
                               unit_generation_opts=_unit_opts())
    assert len(texts) == 1 and len(speech.units) == 1 and speech.audio_wavs[0].dim() == 3
    del tr, m


def _score(uo, enc, ids):
    """The oracle's length-normalised score of hypothesis `ids` (prefix included) over one row's encoder output."""
    ids = torch.tensor(ids)[None]
    lp = torch.log_softmax(uo.project(uo.decoder(uo.embed_text(ids[:, :-1], 0), enc, None)).float(), -1)[0]
    return sum(float(lp[t, ids[0, t + 1]]) for t in range(ids.shape[1] - 1)) / (ids.shape[1] - 1)


def _same_or_near_tie(uo, enc, got, ref_best):
    """Same hypothesis, or a near tie under the oracle's own scoring (test_v1_s2st._audit)."""
    if got == ref_best[1]:
        return True
    assert abs(_score(uo, enc, got) - ref_best[0]) < 2e-2, (got, ref_best)
    return False


WAVES = (32000, 21000)


def _oracle_batch(uo, waves, lang):
    """The oracle's text search over the same zero-padded fbank batch the device runs, with the rows' frame counts.  The
    adaptor's strided conv does not mask padded frames (ASSUMPTIONS.md #8, in the reference and here), so the last
    adaptor frame of the short row depends on the padded Conformer outputs beside it: a row of a ragged batch is not the
    row alone, and the oracle has to see the batch.  Returns the oracle's output and, per row, its unpadded encoder
    output."""
    from oracle.unity_oracle import fbank as o_fbank
    frames = [1 + (n - 400) // 160 for n in WAVES]
    fb = torch.zeros(len(WAVES), max(frames) + max(frames) % 2, 80)
    for b, n in enumerate(WAVES):
        f = o_fbank(waves[b, :n])
        fb[b, :f.shape[0]] = f
    ref = uo.generate(fb, torch.tensor(frames), lang, hard_max=20, output_units=False)
    return ref, [ref["enc"][b:b + 1, :int(ref["enc_lens"][b])] for b in range(len(WAVES))]


@gpu
def test_s2st_matches_oracle(medium):
    """Translator.predict S2ST on a ragged batch (2 s and 1.3 s) against the oracle on the same padded batch: each row's
    text is the oracle's, or an audited near tie; from that text, the oracle's teacher-forced decoder states, T2U encoder
    and unit search give the device's unit hypothesis (up to an audited near tie); EOS ends one row's unit search before
    the budget, so the rows reach the vocoder with different unit counts; each waveform is the fp32 vocoder's on its
    units within 5e-3."""
    from test_v1_s2st import _prefix
    from test_vocoder_durations import oracle_resynth
    cfg, uo, ou, tr = medium["cfg"], medium["uo"], medium["ou"], medium["tr"]
    waves = S.make_waveforms(2, WAVES[0], seed=77)
    texts, speech = tr.predict(tr.fbank_batch(waves, torch.tensor(WAVES)), "s2st", "spa", text_generation_opts=_text_opts(),
                               unit_generation_opts=_unit_opts())
    gen = tr._tls.generator
    text_hyps, unit_hyps = gen.last_text_output.hypotheses, gen.last_unit_output["hypotheses"]
    ref, encs = _oracle_batch(uo, waves, "spa")
    tk = tr.unit_tokenizer
    spkr = C.vocoder_lang_spkr_idx_map("vocoder_36langs")["multispkr"]["spa"][0]
    exact = 0
    for b in range(len(WAVES)):
        ids = text_hyps[b][0][1]
        exact += _same_or_near_tie(uo, encs[b], ids, ref["hyps"][b][0])
        dec = uo.decoder(uo.embed_text(torch.tensor(ids[:-1])[None], 0), encs[b], None)
        t2u_enc = uo.t2u_encoder(dec, None)
        uref = ou.beam_search(t2u_enc, None, _prefix(cfg), beam=5, soft_max=(25, 50), hard_max=40)[0][0]
        got = unit_hyps[b][0]
        if _same_or_near_tie(ou, t2u_enc, got[1], uref):
            # the same hypothesis: its score within fp16 accumulation of the oracle's
            assert abs(got[0] - uref[0]) < 2e-2 + 5e-3 * abs(uref[0]), (got[0], uref[0])
        assert got[1][-1] == cfg.unit_eos, b
        units = tk.create_decoder()(torch.tensor(got[1])[None])[:, 1:]
        assert speech.units[b] == units[0][units[0] != 1].tolist()
        wav, _, _ = oracle_resynth(medium["vc"], medium["vsd"], units, [C.VOCODER_LANGS_V2.index("spa")], [spkr])
        keep = int(wav.shape[-1] * len(speech.units[b]) / units.shape[1])
        out = speech.audio_wavs[b]
        assert out.shape == (1, 1, keep)
        assert (out[0].cpu() - wav[0, :, :keep]).abs().max() < 5e-3, b
    lens = [len(h[0][1]) for h in unit_hyps]
    assert min(lens) < 40 and len(set(lens)) > 1, lens  # EOS won before the forced last step in one row
    print(f"medium s2st: {exact} of {len(WAVES)} texts identical to the oracle's; unit lengths {lens}")


@gpu
@pytest.mark.parametrize("task,lang", [("s2tt", "fra"), ("asr", "eng")])
def test_s2tt_and_asr_match_oracle(medium, task, lang):
    """S2TT and ASR on a ragged batch against the oracle on the same padded batch: the oracle's texts, or audited near
    ties."""
    uo, tr = medium["uo"], medium["tr"]
    waves = S.make_waveforms(2, WAVES[0], seed=13)
    texts, _ = tr.predict(tr.fbank_batch(waves, torch.tensor(WAVES)), task, lang, text_generation_opts=_text_opts())
    hyps = tr._tls.generator.last_text_output.hypotheses
    ref, encs = _oracle_batch(uo, waves, lang)
    for b in range(len(WAVES)):
        assert hyps[b][0][1][:2] == [medium["cfg"].text_eos, medium["toks"][0].lang_index(lang)]
        if _same_or_near_tie(uo, encs[b], hyps[b][0][1], ref["hyps"][b][0]):
            assert texts[b] == ref["texts"][b]


def _runs(tr, waves, ngram=False):
    from seamless_communication_b200.inference import NGramRepeatBlockProcessor
    src = tr.fbank_batch(waves, torch.tensor(WAVES))
    kw = dict(step_processor=NGramRepeatBlockProcessor(2)) if ngram else {}
    return [tr.predict(src, "s2tt", "spa", text_generation_opts=_text_opts(**kw)),
            tr.predict(src, "s2st", "spa", text_generation_opts=_text_opts(**kw), unit_generation_opts=_unit_opts(**kw))]


def _same(a, b):
    (t0, s0), (t1, s1) = a, b
    assert t0 == t1
    if s0 is None:
        assert s1 is None
        return
    assert s0.units == s1.units
    assert len(s0.audio_wavs) == len(s1.audio_wavs) and all(torch.equal(x, y) for x, y in zip(s0.audio_wavs, s1.audio_wavs))


@gpu
def test_fp8_equals_fp16_on_dequantized(medium):
    """decoder_weight_dtype=float8_e4m3fn on medium (text search and AR unit search on e4m3 weights): S2TT and S2ST,
    with and without n-gram blocking, equal an fp16 model of dequantize_decoder_weights(sd) bit for bit."""
    from seamless_communication_b200.inference import Translator
    from seamless_communication_b200.models.fp8_weights import dequantize_decoder_weights
    from seamless_communication_b200.models.unity import load_unity_model
    cfg, sd, toks, voc = medium["cfg"], medium["sd"], medium["toks"], medium["voc"]
    waves = S.make_waveforms(2, WAVES[0], seed=21)
    f8 = load_unity_model("seamlessM4T_medium", state_dict=sd, tokenizers=toks, decoder_weight_dtype=torch.float8_e4m3fn)
    assert f8.engine.fp8 and f8.t2u_model.unit_engine.fp8
    a = [r for ng in (False, True) for r in _runs(Translator(f8, voc, device="cuda:0"), waves, ng)]
    del f8
    f16 = load_unity_model("seamlessM4T_medium", state_dict=dequantize_decoder_weights(sd, cfg), tokenizers=toks)
    b = [r for ng in (False, True) for r in _runs(Translator(f16, voc, device="cuda:0"), waves, ng)]
    del f16
    for x, y in zip(a, b):
        _same(x, y)


@gpu
def test_two_lanes_equal_serial(medium):
    """Two LanePool lanes bound to both engines of medium give the serial S2ST results bit for bit."""
    from seamless_communication_b200.parallel import LanePool
    tr, model = medium["tr"], medium["model"]

    def run(w):
        return tr.predict(tr.fbank_batch(w), "s2st", "spa", text_generation_opts=_text_opts(), unit_generation_opts=_unit_opts())
    batches = [S.make_waveforms(2, 24000, seed=s) for s in (5, 6, 7)]
    serial = [run(w) for w in batches]
    pool = LanePool("cuda", 2, model.engines)
    try:
        par = pool.map(run, [[w] for w in batches])
    finally:
        pool.close()
    for x, y in zip(serial, par):
        _same(x, y)


@gpu
def test_fairseq_checkpoint_gives_same_translations(medium):
    """load_unity_model("seamlessM4T_medium", checkpoint=<fairseq-named checkpoint of the same weights>): the text
    encoder is dropped, the unit engine is built from the AR T2U keys, and the texts, units and waveforms equal the
    state-dict model's."""
    from seamless_communication_b200.inference import Translator
    from seamless_communication_b200.models.unity import load_unity_model
    m = load_unity_model("seamlessM4T_medium", checkpoint=fairseq_medium_checkpoint(medium["sd"]), tokenizers=medium["toks"])
    a, b = m.t2u_model.unit_engine.w, medium["model"].t2u_model.unit_engine.w
    assert sorted(a) == sorted(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert not any(k.startswith("text_encoder") for k in m.engine.w)
    waves = S.make_waveforms(2, WAVES[0], seed=31)
    got = _runs(Translator(m, medium["voc"], device="cuda:0"), waves)
    del m
    want = _runs(medium["tr"], waves)
    for x, y in zip(got, want):
        _same(x, y)
