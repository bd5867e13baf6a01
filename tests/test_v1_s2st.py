"""Speech output for seamlessM4T_large (v1): the autoregressive T2U (t2u_builder.py:311-427) as a unit beam search on the
text decoder's step kernels, and the vocoder_36langs card.

The AR T2U decoder is the NLLB decoder type over the unit vocabulary, so its oracle is `UnityOracle.decoder` /
`beam_search` (pinned against the reference's C++ mirror) over the renamed weights (`t2u_decoder_state_dict`) and the
derived config (`t2u_decoder_config`); the T2U encoder is `UnityOracle.t2u_encoder`.  CPU tests cover the config, the
synthetic and fairseq names, the renaming, the vocoder card and the error paths; GPU tests hold the device path to the
oracle and to its own batch / bucket / lane invariants."""
import dataclasses
import json
import os
import types

import pytest
import torch

from oracle.unity_oracle import UnityOracle, fbank as o_fbank, key_mask
from oracle_v1 import UnityOracleV1
from seamless_communication_b200 import config as C, synthetic as S
from seamless_communication_b200.inference.generator import filter_unit_ngrams, remove_consecutive_repeated_ngrams
from seamless_communication_b200.models import checkpoint as ck
from seamless_communication_b200.models.unity.model import t2u_decoder_config, t2u_decoder_state_dict
from seamless_communication_b200.models.unity import UnitTokenizer

G = os.path.join(os.path.dirname(__file__), "golden")
dev = "cuda"
gpu = pytest.mark.gpu


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-9)).item()


def ar_state_dict(arch="tiny_v1", seed=0):
    return S.make_unity_state_dict(C.UNITY_ARCHS[arch](), seed, dec_gain=4.0, with_t2u=True)


def unit_oracle(cfg, sd):
    """The AR T2U decoder / unit beam search of the reference, as the text decoder's oracle over the renamed weights."""
    return UnityOracle(t2u_decoder_config(cfg).to_dict(), t2u_decoder_state_dict(sd))


# ------------------------------------------------------------------------------------------------ CPU
def test_ar_t2u_config():
    b = C.base()
    assert (b.t2u_enc_layers, b.t2u_dec_layers, b.t2u_ffn_dim, b.num_heads, b.unit_vocab, b.unit_max_seq_len) == \
           (6, 6, 8192, 16, 10082, 2048)
    assert (b.unit_bos, b.unit_pad, b.unit_eos, b.unit_unk) == (0, 1, 2, 3)
    for arch in ("base", "tiny_v1", "small_v1"):
        c = C.UNITY_ARCHS[arch]()
        assert c.unit_vocab == c.num_units + 2 * (len(c.unit_langs) + 1) + 4 == UnitTokenizer(c.num_units, c.unit_langs, arch).vocab_info.size
        d = t2u_decoder_config(c)
        assert (d.dec_layers, d.dec_ffn_dim, d.text_vocab, d.max_seq_len) == (c.t2u_dec_layers, c.t2u_ffn_dim, c.unit_vocab, 2048)
        assert (d.text_bos, d.text_pad, d.text_eos, d.text_unk) == (0, 1, 2, 3)
        assert (d.model_dim, d.num_heads) == (c.model_dim, c.num_heads)


def test_ar_t2u_synthetic_keys_and_text_part_unchanged():
    cfg = C.tiny_v1()
    sd, plain = ar_state_dict(), S.make_unity_state_dict(cfg, 0, dec_gain=4.0)
    assert set(plain) <= set(sd) and all(torch.equal(plain[k], sd[k]) for k in plain)
    t2u = sorted(k for k in sd if k not in plain)
    assert all(k.startswith("t2u_model.") for k in t2u)
    M, F = cfg.model_dim, cfg.t2u_ffn_dim
    for k, shape in (("t2u_model.encoder.layers.0.self_attn.q_proj.weight", (M, M)),
                     ("t2u_model.encoder.layers.0.ffn.inner_proj.weight", (F, M)), ("t2u_model.encoder.layer_norm.bias", (M,)),
                     ("t2u_model.decoder_frontend.embed.weight", (cfg.unit_vocab, M)),
                     (f"t2u_model.decoder.layers.{cfg.t2u_dec_layers - 1}.encoder_decoder_attn.v_proj.weight", (M, M)),
                     ("t2u_model.decoder.layers.0.encoder_decoder_attn_layer_norm.weight", (M,)),
                     ("t2u_model.decoder.layers.1.ffn.output_proj.weight", (M, F)), ("t2u_model.decoder.layer_norm.weight", (M,))):
        assert sd[k].shape == shape, k
    assert sd["t2u_model.final_proj.weight"] is sd["t2u_model.decoder_frontend.embed.weight"]  # TiedProjection (:323)
    assert not any("embed_char" in k or "conv1d" in k or "variance_adaptor" in k for k in t2u)
    assert len([k for k in t2u if k.startswith("t2u_model.encoder.layers.")]) == cfg.t2u_enc_layers * 16
    assert len([k for k in t2u if k.startswith("t2u_model.decoder.layers.")]) == cfg.t2u_dec_layers * 26


def test_t2u_renaming_consumes_every_ar_key_exactly_once():
    """Every AR T2U key goes either to the T2U encoder (kept under its own name) or, renamed, to exactly one parameter of
    the decoder-only engine, and the renamed set is exactly the text decoder's parameter set at the derived config."""
    for arch in ("tiny_v1", "small_v1"):
        cfg = C.UNITY_ARCHS[arch]()
        sd = ar_state_dict(arch)
        ar = {k for k in sd if k.startswith("t2u_model.")}
        enc = {k for k in ar if k.startswith("t2u_model.encoder.")}
        dec = t2u_decoder_state_dict(sd)
        consumed = [k for k in ar - enc for v in dec.values() if v is sd[k]]
        # the tied projection and embedding are one tensor: both names map to it
        assert sorted(set(consumed)) == sorted(ar - enc) and len(dec) == len(ar - enc)
        want = S.make_unity_state_dict(dataclasses.replace(t2u_decoder_config(cfg), encoder_variant="v2"), 0, with_t2u=False)
        want = {k: v for k, v in want.items() if k.startswith(("text_decoder", "final_proj"))}
        assert sorted(dec) == sorted(want)
        assert all(dec[k].shape == want[k].shape for k in want)
        assert not any(k.startswith("t2u_model.") for k in dec)


_ENC_LAYER = [("self_attn.output_proj.", "self_attn.out_proj."), ("ffn.inner_proj.", "fc1."), ("ffn.output_proj.", "fc2."),
              ("ffn_layer_norm.", "final_layer_norm."), ("", "")]
_DEC_LAYER = [("encoder_decoder_attn.output_proj.", "encoder_attn.out_proj."),
              ("encoder_decoder_attn_layer_norm.", "encoder_attn_layer_norm."), ("encoder_decoder_attn.", "encoder_attn.")] + _ENC_LAYER


def ar_to_fairseq(key):
    """fairseq2 name of an AR T2U parameter -> its name in the original fairseq checkpoint."""
    fixed = {"t2u_model.encoder.layer_norm.": "synthesizer_encoder.layer_norm.", "t2u_model.decoder.layer_norm.": "decoder.layer_norm.",
             "t2u_model.decoder_frontend.embed.": "decoder.embed_tokens.", "t2u_model.final_proj.": "decoder.output_projection."}
    for a, b in fixed.items():
        if key.startswith(a):
            return b + key[len(a):]
    parts = key.split(".")
    src, table = ("synthesizer_encoder", _ENC_LAYER) if parts[1] == "encoder" else ("decoder", _DEC_LAYER)
    rest = ".".join(parts[4:])
    for a, b in table:
        if rest.startswith(a):
            return f"{src}.layers.{parts[3]}." + b + rest[len(a):]
    raise KeyError(key)


def fairseq_ar_checkpoint(sd):
    """A fairseq-named v1 checkpoint with the AR T2U (decoder.*, synthesizer_encoder.*, both tied tables present, as in
    the release) that convert_unity_checkpoint turns back into `sd`."""
    from test_v1_encoder import to_fairseq
    fs = {(ar_to_fairseq(k) if k.startswith("t2u_model.") else to_fairseq(k)): v.clone() for k, v in sd.items()
          if k != "text_decoder_frontend.embed.weight"}
    emb = sd["final_proj.weight"].clone()
    emb[[1, 3, 0, 2]] = sd["final_proj.weight"][[0, 1, 2, 3]]
    fs["target_letter_decoder.output_projection.weight"] = emb
    fs["decoder.version"] = torch.tensor([3.0])
    return {"model": fs}


def test_fairseq_v1_checkpoint_with_ar_t2u_converts():
    """The fairseq checkpoint converts back to the synthetic fairseq2 state dict, unit embedding and projection tied."""
    sd = ar_state_dict()
    out = ck.convert_unity_checkpoint(fairseq_ar_checkpoint(sd), nllb_vocab=C.tiny_v1().text_vocab)["model"]
    assert sorted(out) == sorted(sd)
    for k in sd:
        assert torch.equal(out[k], sd[k]), k
    assert out["t2u_model.decoder_frontend.embed.weight"] is out["t2u_model.final_proj.weight"]


def test_vocoder_36langs_card_matches_reference():
    """The card's language / speaker table (tests/golden/vocoder_36langs_map.json, made from the reference card by
    make_golden_vocoder36.py): same languages as vocoder_v2, its own first speakers."""
    d = json.load(open(os.path.join(G, "vocoder_36langs_map.json")))
    assert C.VOCODER_CARDS["vocoder_36langs"] == d["model_arch"] == "base"
    ref = d["lang_spkr_idx_map"]
    m = C.vocoder_lang_spkr_idx_map("vocoder_36langs")
    assert m["multilingual"] == ref["multilingual"]
    assert m["multispkr"] == {lang: spk[:1] for lang, spk in ref["multispkr"].items()}
    assert m["multispkr"]["ben"] == [2] and m["multispkr"]["cmn"] == [5]
    assert C.vocoder_lang_spkr_idx_map()["multispkr"]["ben"] == [1]  # vocoder_v2 unchanged


def test_unit_ngram_filtering_is_batch_one_only():
    u = torch.tensor([[9, 4, 4, 5, 6, 5, 6, 1]])
    assert filter_unit_ngrams(u).tolist() == [remove_consecutive_repeated_ngrams(u[0].tolist())] == [[9, 4, 5, 6, 1]]
    with pytest.raises(NotImplementedError, match="batch_size > 1"):
        filter_unit_ngrams(torch.cat([u, u]))


def test_t2st_on_v1_still_raises():
    """Text input needs the NLLB text encoder: T2ST on a v1 model raises even when its AR T2U is loaded."""
    from seamless_communication_b200.inference import Translator
    tr = Translator.__new__(Translator)
    tr.model, tr.apply_mintox = types.SimpleNamespace(config=C.tiny_v1(), t2u_model=object()), False
    with pytest.raises(NotImplementedError, match="text input"):
        tr.predict(torch.zeros(4), "t2st", "spa", src_lang="eng")
    tr.model = types.SimpleNamespace(config=C.tiny_v1(), t2u_model=None)
    with pytest.raises(NotImplementedError, match="AR T2U"):
        tr.predict(torch.zeros(4), "s2st", "spa")


# ------------------------------------------------------------------------------------------------ GPU
def with_reachable_eos(sd, cfg, scale=3.0, seed=11):
    """The synthetic T2U scores EOS 0, so every search runs to its budget.  An EOS row `scale` times the other rows'
    spread makes some unit searches end early (on the inputs below: 7, 11, 31 and 40 units of 40), so EOS termination
    and ragged unit lengths reach the vocoder."""
    e = sd["t2u_model.final_proj.weight"].clone()
    g = torch.Generator().manual_seed(seed)
    e[cfg.unit_eos] = (torch.randn(cfg.model_dim, generator=g) * scale * 0.25 * cfg.model_dim ** -0.5).half().float()
    return {**sd, "t2u_model.final_proj.weight": e, "t2u_model.decoder_frontend.embed.weight": e}


@pytest.fixture(scope="module")
def tiny():
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    cfg, vc = C.tiny_v1(), C.tiny_vocoder()
    sd = with_reachable_eos(ar_state_dict(), cfg)
    toks = S.make_tokenizers(cfg)
    vsd = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
    return dict(cfg=cfg, sd=sd, toks=toks, vc=vc, vsd=vsd, model=load_unity_model("tiny_v1", state_dict=sd, tokenizers=toks),
                voc=load_vocoder_model("tiny", state_dict=vsd), uo=UnityOracleV1(cfg.to_dict(), sd, toks), ou=unit_oracle(cfg, sd))


def _states(B, L, M, seed, lens):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, M, generator=g).half().float()
    for b in range(B):
        x[b, lens[b]:] = 0
    return x


def _prefix(cfg, lang="spa"):
    return UnitTokenizer(cfg.num_units, cfg.unit_langs, cfg.name).create_encoder(lang).prefix_indices.tolist()


@gpu
@pytest.mark.parametrize("arch", ["tiny_v1", "small_v1"])
def test_t2u_encoder_and_teacher_forced_logits_match_oracle(arch, tiny):
    """T2U encoder output and teacher-forced unit logits (decode + project) against the fp32 oracle on a ragged batch,
    tolerances as test_v1_encoder.py: max error over max |ref| below 5e-3 on the valid rows."""
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.nn import PaddingMask
    if arch == "tiny_v1":
        cfg, sd, t2u = tiny["cfg"], tiny["sd"], tiny["model"].t2u_model
    else:
        cfg, sd = C.small_v1(), ar_state_dict("small_v1", 5)
        t2u = load_unity_model("small_v1", state_dict=sd, tokenizers=S.make_tokenizers(cfg)).t2u_model
    M, lens = cfg.model_dim, [23, 9]
    x = _states(2, 23, M, 1, lens)
    mask = PaddingMask(torch.tensor(lens), 23)
    enc, _ = t2u.encode(x.to(dev).half(), mask)
    uo = UnityOracleV1(cfg.to_dict(), sd)
    km = key_mask(torch.tensor(lens), 23)
    o_enc = uo.t2u_encoder(x, km)
    for b in range(2):
        assert rel(enc[b, :lens[b]], o_enc[b, :lens[b]]) < 5e-3, b
    g = torch.Generator().manual_seed(2)
    seqs = torch.cat([torch.tensor(_prefix(cfg))[None].expand(2, -1),
                      torch.randint(4, cfg.num_units + 4, (2, 40), generator=g)], 1)
    dec, _ = t2u.decode(seqs.to(dev), None, enc, mask)
    logits = t2u.project(dec, None).logits
    ou = unit_oracle(cfg, sd)
    o_logits = ou.project(ou.decoder(ou.embed_text(seqs, 0), o_enc, km))
    assert logits.shape == (2, 42, cfg.unit_vocab) and torch.isfinite(logits).all()
    assert rel(logits, o_logits) < 5e-3


def _audit(ou, enc_b, hyp, ref_best):
    """Same hypothesis, or a near tie under the oracle's own scoring (ASSUMPTIONS.md #9)."""
    if hyp[1] == ref_best[1]:
        return
    ids = torch.tensor(hyp[1])[None]
    lp = torch.log_softmax(ou.project(ou.decoder(ou.embed_text(ids[:, :-1], 0), enc_b, None)).float(), -1)[0]
    sc = sum(float(lp[t, ids[0, t + 1]]) for t in range(ids.shape[1] - 1)) / (ids.shape[1] - 1)
    assert abs(sc - ref_best[0]) < 2e-2, (sc, ref_best[0])


@gpu
def test_unit_search_matches_oracle(tiny):
    """The unit beam search on the oracle's own T2U encoder output (rounded to fp16) gives the oracle's hypotheses."""
    cfg, ou, t2u = tiny["cfg"], tiny["ou"], tiny["model"].t2u_model
    from seamless_communication_b200.ops import Seq
    lens = [11, 6]
    x = _states(2, 11, cfg.model_dim, 3, lens)
    o_enc = tiny["uo"].t2u_encoder(x, key_mask(torch.tensor(lens), 11)).half()
    for b in range(2):
        o_enc[b, lens[b]:] = 0
    prefix = _prefix(cfg)
    ref = ou.beam_search(o_enc.float(), torch.tensor(lens), prefix, beam=5, soft_max=(25, 50), hard_max=48)
    e = Seq(2, 11, cfg.model_dim, buf=o_enc.to(dev).view(22, -1))
    hyps = t2u.beam_search(e, torch.tensor(lens, dtype=torch.int32, device=dev), prefix, beam=5, soft_max=(25, 50), hard_max=48)
    for b in range(2):
        assert hyps[b][0][1][:2] == prefix
        _audit(ou, o_enc[b:b + 1, :lens[b]].float(), hyps[b][0], ref[b][0])


@gpu
def test_long_unit_search_harvests_decode_full_states_on_both_chains():
    """A 700-position unit search on small_v1 (full width, 10 082 units, 79 projection tiles) on the default step chain
    and with SB_DECODE_GEMM_T=0: the states harvested from the search equal decode_full over the winning hypotheses at
    positions < 128, >= 128 and >= 512 (5e-3 of max |ref|), both chains find the same hypotheses, and each run is
    bit-identical when repeated."""
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.ops import Seq
    cfg = C.small_v1()
    t2u = load_unity_model("small_v1", state_dict=ar_state_dict("small_v1", 6), tokenizers=S.make_tokenizers(cfg)).t2u_model
    eng, M, lens = t2u.unit_engine, cfg.model_dim, [27, 16]
    enc = Seq(2, 27, M, buf=_states(2, 27, M, 4, lens).view(54, M).to(dev).half())
    el = torch.tensor(lens, dtype=torch.int32, device=dev)
    prefix = _prefix(cfg)
    runs = {}
    for gemm_t in (True, False):
        eng.decode_gemm_t = gemm_t
        try:
            out = []
            for _ in range(2):
                hyps = t2u.beam_search(enc, el, prefix, beam=5, soft_max=(25, 50), hard_max=700)
                best = [h[0][1] for h in hyps]
                st = eng.harvest_decoder_states([len(s) - 1 for s in best])
                out.append((hyps, st.buf.view(2, -1, M).clone()))
        finally:
            eng.decode_gemm_t = True
        assert out[0][0] == out[1][0] and torch.equal(out[0][1], out[1][1]), gemm_t
        runs[gemm_t] = out[0]
    assert runs[True][0] == runs[False][0]
    hyps, harvested = runs[True]
    best = [h[0][1] for h in hyps]
    assert all(len(s) == 700 for s in best)
    seqs = torch.tensor([s[:-1] for s in best], device=dev)
    full = eng.decode_full(seqs, torch.full((2,), 699, dtype=torch.int32, device=dev), enc, el).buf.view(2, -1, M)
    for lo, hi in ((0, 128), (128, 512), (512, 699)):
        assert rel(harvested[:, lo:hi], full[:, lo:hi]) < 5e-3, (lo, hi)


def _oracle_s2st(tiny, wave, lang, text_hard, unit_hard):
    """fp32 reference chain of Translator.predict(wave, "s2st") for one utterance: text search, teacher-forced decoder
    states, T2U encoder, unit search, UnitTokenDecoder, lang token dropped, vocoder with duration prediction, trim."""
    from test_vocoder_durations import oracle_resynth
    cfg, uo, ou = tiny["cfg"], tiny["uo"], tiny["ou"]
    fb = o_fbank(wave)
    fb = torch.cat([fb, torch.zeros(fb.shape[0] % 2, 80)])[None]
    out = uo.generate(fb, None, lang, hard_max=text_hard, output_units=False)
    ids = out["text_ids"][0]
    ts = torch.tensor(ids[:-1])[None]
    dec = uo.decoder(uo.embed_text(ts, 0), out["enc"], None)
    t2u_enc = uo.t2u_encoder(dec, None)
    hyp = ou.beam_search(t2u_enc, None, _prefix(cfg, lang), beam=5, soft_max=(25, 50), hard_max=unit_hard)[0][0]
    tk = UnitTokenizer(cfg.num_units, cfg.unit_langs, cfg.name)
    units = tk.create_decoder()(torch.tensor(hyp[1])[None])[:, 1:]
    speech_units = units[0][units[0] != 1].tolist()
    vlang = C.VOCODER_LANGS_V2.index(lang)
    wav, _, _ = oracle_resynth(tiny["vc"], tiny["vsd"], units, [vlang], [C.vocoder_lang_spkr_idx_map()["multispkr"][lang][0]])
    n = int(wav.shape[-1] * len(speech_units) / units.shape[1])
    return ids, speech_units, wav[0, :, :n], t2u_enc, hyp


@gpu
def test_translator_s2st_tiny_v1_matches_oracle(tiny):
    """Translator.predict(wave, "s2st") on tiny_v1 + a tiny vocoder with a duration predictor: the oracle's text, its
    unit hypothesis (ended by EOS before the budget) and units, and its waveform within test_vocoder_durations.py's
    5e-3."""
    from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator
    tr = Translator(tiny["model"], tiny["voc"], device="cuda:0")
    wave = S.make_waveforms(2, 32000, seed=77)[0]
    texts, speech = tr.predict(wave, "s2st", "spa", text_generation_opts=SequenceGeneratorOptions(hard_max_seq_len=20),
                               unit_generation_opts=SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40))
    ids, units, wav, t2u_enc, hyp = _oracle_s2st(tiny, wave, "spa", 20, 40)
    gen = Translator._last_generator
    assert gen.last_text_output.hypotheses[0][0][1] == ids
    got_hyp = gen.last_unit_output["hypotheses"][0][0]
    assert got_hyp[1] == hyp[1] and abs(got_hyp[0] - hyp[0]) < 2e-2
    assert len(hyp[1]) < 40 and hyp[1][-1] == tiny["cfg"].unit_eos  # EOS won before the forced last step
    assert speech.units[0] == units and len(units) > 0
    got = speech.audio_wavs[0]
    assert got.shape == (1, 1, wav.shape[-1])
    assert (got[0].cpu() - wav).abs().max() < 5e-3


def _predict(tr, waves, ns=None):
    from seamless_communication_b200.inference import SequenceGeneratorOptions
    src = tr.fbank_batch(waves, None if ns is None else torch.tensor(ns))
    return tr.predict(src, "s2st", "spa", text_generation_opts=SequenceGeneratorOptions(hard_max_seq_len=20),
                      unit_generation_opts=SequenceGeneratorOptions(soft_max_seq_len=(25, 50), hard_max_seq_len=40))


@gpu
def test_ragged_batch_rows_equal_rows_alone(tiny):
    """In a ragged batch through Translator.predict, EOS ends the unit rows at different lengths, and from the T2U
    encoder output on, every row gives the hypotheses, the units and, bit for bit, the samples of that row run alone:
    the row's own T2U encoder rows searched alone, its units vocoded alone and trimmed by its own length.  (The speech
    encoder agrees with a row encoded alone to fp16 rounding only, test_small_v1_rows_independent_and_deterministic.)"""
    from seamless_communication_b200.inference import Translator
    from seamless_communication_b200.ops import Seq
    tr = Translator(tiny["model"], tiny["voc"], device="cuda:0")
    t2u, cfg = tiny["model"].t2u_model, tiny["cfg"]
    ns = [32000, 24011, 17000]
    waves = S.make_waveforms(3, 32000, seed=91)
    texts, speech = _predict(tr, waves, ns)
    out = Translator._last_generator.last_unit_output
    hyps, enc = out["hypotheses"], out["t2u_enc"]
    n_units = [len(h[0][1]) for h in hyps]
    assert len(set(n_units)) > 1 and min(n_units) < 40, n_units  # EOS ended rows at different lengths
    L, M = enc.T, cfg.model_dim
    for b in range(3):
        n = int(enc.lens[b])
        e = Seq(1, L, M, buf=enc.buf.view(3, L, M)[b].contiguous())
        alone = t2u.beam_search(e, enc.lens[b:b + 1], _prefix(cfg), beam=5, soft_max=(25, 50), hard_max=40)
        assert [h[1] for h in alone[0]] == [h[1] for h in hyps[b]], (b, n)
        row = torch.tensor(hyps[b][0][1])[None]  # the generator's input to UnitTokenDecoder for this row alone
        units = tr.unit_tokenizer.create_decoder()(row)
        s1 = tr._speech_output_ar(units, [units.shape[1]], "spa", -1, 16000)
        assert s1.units[0] == speech.units[b]
        assert torch.equal(s1.audio_wavs[0], speech.audio_wavs[b]), b
    # output assembly with unit rows of different lengths (a genuine unit 1 included): each row as the row alone
    vc, voc = tiny["vc"], tiny["voc"]
    lang = 6000  # any decoded language symbol: it is dropped
    rows = [[lang, 9, 1, 33, 7, 1], [lang, 4, 4, 5, 1], [lang, 17, 1]]
    units = torch.ones(3, 6, dtype=torch.int64)
    for b, r in enumerate(rows):
        units[b, :len(r)] = torch.tensor(r)
    out = tr._speech_output_ar(units, [len(r) for r in rows], "spa", -1, 16000)
    for b, r in enumerate(rows):
        u = torch.tensor(r[1:], device=dev)[None]
        w = voc(u, "spa", -1)
        keep = int(int(voc.last_wav_lens[0]) * len([x for x in r[1:] if x != 1]) / len(r[1:]))
        assert out.units[b] == [x for x in r[1:] if x != 1]
        assert torch.equal(out.audio_wavs[b], w[:, :, :keep]), b


@gpu
def test_bucketed_encoder_length_equals_unbucketed(tiny):
    """Under the translator's unit options (soft (25, 50), hard_max 1024), two short text lengths of one bucket, whose
    length budgets (175 and 275) differ, search on one cached state and its graphs, and give the hypotheses of the
    unbucketed search (unpadded encoder rows, state sized by the budget).  Lengths may also be left out."""
    from seamless_communication_b200.ops import Seq
    cfg, t2u = tiny["cfg"], tiny["model"].t2u_model
    M, prefix = cfg.model_dim, _prefix(cfg)
    eng = t2u.unit_engine
    new_keys = []
    for S_, lens in ((5, [5, 3]), (9, [9, 9]), (9, None)):
        enc = Seq(2, S_, M, buf=_states(2, S_, M, S_, lens or [S_, S_]).view(2 * S_, M).to(dev).half())
        el = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
        before = set(eng._graphs)
        a = t2u.beam_search(enc, el, prefix, soft_max=(25, 50), hard_max=1024, bucket=True)
        new_keys.append(set(eng._graphs) - before)
        b = t2u.beam_search(enc, el, prefix, soft_max=(25, 50), hard_max=1024, bucket=False)
        assert [[h[1] for h in r] for r in a] == [[h[1] for h in r] for r in b]
        assert all(abs(x[0] - y[0]) < 1e-4 for ra, rb in zip(a, b) for x, y in zip(ra, rb))
    # the cache key starts (B, S_enc, allocated length): one new state of 32 rows x 1024 positions, then none
    assert [k[:3] for k in new_keys[0]] == [(2, 32, 1024)] and not new_keys[1] and not new_keys[2]


@gpu
def test_vocoder_splits_batches_past_one_gemm_grid(tiny):
    """A duration-predicted batch whose frames exceed one sb_gemm grid is generated in halves: same samples, bit for
    bit, and the same lengths as one pass (the limit is lowered on the instance to reach it at test size)."""
    vc, voc = tiny["vc"], tiny["voc"]
    eng = voc.code_generator
    g = torch.Generator().manual_seed(4)
    units = torch.randint(0, vc.num_embeddings, (5, 23), generator=g).to(dev)
    one, lens1, dur1 = eng.resynthesize(units, [3] * 5, [7] * 5)
    eng.MAX_GEMM_ROWS = int(units.shape[0] * lens1.max() // vc.hop * eng._max_rate() // 3)
    try:
        split, lens2, dur2 = eng.resynthesize(units, [3] * 5, [7] * 5)
    finally:
        del eng.MAX_GEMM_ROWS
    assert torch.equal(lens1, lens2) and torch.equal(dur1, dur2)
    assert torch.equal(one, split)


@gpu
def test_two_lanes_equal_serial(tiny):
    """Two LanePool lanes bound to both engines (model.engines) give the serial results, units and samples bit for bit."""
    from seamless_communication_b200.inference import Translator
    from seamless_communication_b200.parallel import LanePool
    tr = Translator(tiny["model"], tiny["voc"], device="cuda:0")
    batches = [S.make_waveforms(2, 24000, seed=s) for s in (5, 6, 7)]
    serial = [_predict(tr, w) for w in batches]
    assert len(tiny["model"].engines) == 2
    pool = LanePool("cuda", 2, tiny["model"].engines)
    try:
        par = pool.map(lambda w: _predict(tr, w), [[w] for w in batches])
    finally:
        pool.close()
    for (t0, s0), (t1, s1) in zip(serial, par):
        assert t0 == t1 and s0.units == s1.units
        assert all(torch.equal(a, b) for a, b in zip(s0.audio_wavs, s1.audio_wavs))


@gpu
def test_fairseq_checkpoint_loads_same_unit_engine(tiny):
    from seamless_communication_b200.models.unity import load_unity_model
    m = load_unity_model("tiny_v1", checkpoint=fairseq_ar_checkpoint(tiny["sd"]), tokenizers=tiny["toks"])
    a, b = m.t2u_model.unit_engine.w, tiny["model"].t2u_model.unit_engine.w
    assert sorted(a) == sorted(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert not m.engine.has_t2u and m.engine.has_t2u_encoder
    assert torch.equal(m.engine.w["t2u_model.encoder.layer_norm.w"], tiny["model"].engine.w["t2u_model.encoder.layer_norm.w"])
