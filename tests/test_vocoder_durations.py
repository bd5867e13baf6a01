"""Vocoder duration prediction (CodeGenerator.forward with dur_prediction=True, reference codehifigan.py:75-101).

CPU: the fp32 oracle below against the reference's own output (tests/golden/codehifigan_dur_tiny.npz, made by
tests/golden/make_golden_vocoder_dur.py), and weight loading.  GPU: the device path against the fixture and the oracle,
and exact invariants of the per-row masking that lets one batch hold rows of different lengths."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.unity_oracle import UnityOracle, VocoderOracle
from seamless_communication_b200 import config as C, synthetic as S

G = os.path.join(os.path.dirname(__file__), "golden")
dev = "cuda"
P = "code_generator"


def oracle_resynth(vc, vsd, units, lang, spkr, durations=None):
    """fp32 CodeGenerator.forward(dur_prediction=True): VariancePredictor on dict(units) (padding_mask None),
    dur = clamp(round(exp(l) - 1), 1), each row's [lang | dict | spkr] frames repeated by dur, HiFi-GAN per row.
    Returns (wav (N,1,hop*max T_b) with zeros past each row's end, exp(l) - 1, dur)."""
    vo = VocoderOracle(vc.to_dict(), vsd)
    uo = UnityOracle(C.tiny_v2().to_dict(), vsd)  # only its VariancePredictor / LayerNorm / Linear are used
    x = F.embedding(units, vsd[f"{P}.dict.weight"])  # (N, U, E)
    raw = torch.exp(uo.variance_predictor(x, torch.ones(units.shape, dtype=torch.bool), f"{P}.dur_predictor")) - 1
    dur = torch.clamp(torch.round(raw).long(), min=1) if durations is None else durations.long()
    tot = dur.sum(1)
    wav = torch.zeros(units.shape[0], 1, int(tot.max()) * vc.hop)
    for b in range(units.shape[0]):
        xe = x[b].repeat_interleave(dur[b], dim=0).t()  # (E, T_b)
        T = xe.shape[1]
        lg = vsd[f"{P}.lang.weight"][lang[b]][:, None].expand(-1, T)
        sp = vsd[f"{P}.spkr.weight"][spkr[b]][:, None].expand(-1, T)
        wav[b, :, :T * vc.hop] = vo.generator(torch.cat([lg, xe, sp], 0)[None])[0]
    return wav, raw, dur


# ------------------------------------------------------------------------------------------------ CPU
def test_oracle_matches_reference_fixture():
    d = np.load(os.path.join(G, "codehifigan_dur_tiny.npz"))
    vc = C.tiny_vocoder()
    vsd = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
    for case in ("one", "two"):
        units = torch.from_numpy(d[f"{case}.units"])
        wav, raw, dur = oracle_resynth(vc, vsd, units, d[f"{case}.lang"].tolist(), d[f"{case}.spkr"].tolist())
        assert np.array_equal(dur.numpy(), d[f"{case}.dur"])
        assert np.abs(raw.numpy() - d[f"{case}.raw"]).max() < 1e-5
        assert wav.shape == d[f"{case}.wav"].shape
        assert np.abs(wav.numpy() - d[f"{case}.wav"]).max() < 2e-5
    # the fixture exercises clamped 1s and durations of at least 4
    assert d["one.dur"].min() == 1 and d["one.dur"].max() >= 4


def test_duration_predictor_weights_are_opt_in():
    """Adding the predictor leaves every other synthetic tensor as it was (the existing checksum fixture pins those)."""
    for vc in (C.tiny_vocoder(), C.base_vocoder()):
        a = S.make_vocoder_state_dict(vc, seed=1)
        b = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
        extra = sorted(set(b) - set(a))
        assert set(a) <= set(b) and all(k.startswith(f"{P}.dur_predictor.") for k in extra) and len(extra) == 10
        assert all(torch.equal(a[k], b[k]) for k in a)
        assert b[f"{P}.dur_predictor.conv1.0.weight"].shape == (vc.var_pred_hidden, vc.embedding_dim, vc.var_pred_kernel)


def test_partial_duration_predictor_is_rejected():
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    vc = C.tiny_vocoder()
    sd = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
    for gone in ("ln2.bias", "proj.weight"):
        part = {k: v for k, v in sd.items() if k != f"{P}.dur_predictor.{gone}"}
        with pytest.raises(ValueError, match=gone.replace(".", r"\.")):
            load_vocoder_model("tiny", device="cpu", state_dict=part)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def tiny():
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    vc = C.tiny_vocoder()
    vsd = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
    return vc, vsd, load_vocoder_model("tiny", state_dict=vsd)


def _both_resblock_paths(eng):
    """Runs the body once on the fused ResBlock kernel and once conv by conv (what SB_FUSED_RESBLOCK=0 selects)."""
    for fused in (True, False):
        eng.fused_resblocks = fused
        try:
            yield fused
        finally:
            eng.fused_resblocks = True


@pytest.mark.gpu
def test_tiny_matches_reference_fixture(tiny):
    vc, _, voc = tiny
    eng = voc.code_generator
    d = np.load(os.path.join(G, "codehifigan_dur_tiny.npz"))
    for fused in _both_resblock_paths(eng):
        for case in ("one", "two"):
            units = torch.from_numpy(d[f"{case}.units"]).to(dev)
            langs = [C.VOCODER_LANGS_V2[i] for i in d[f"{case}.lang"].tolist()]
            wav = voc(units, langs, d[f"{case}.spkr"].tolist())  # dur_prediction=True is the default
            _, _, dur = eng.resynthesize(units, d[f"{case}.lang"].tolist(), d[f"{case}.spkr"].tolist())
            assert np.array_equal(dur.cpu().numpy(), d[f"{case}.dur"]), (fused, case)
            assert wav.shape == d[f"{case}.wav"].shape
            err = np.abs(wav.cpu().numpy() - d[f"{case}.wav"]).max()
            assert err < 5e-3, (fused, case, err)
            assert voc.last_wav_lens.tolist() == (d[f"{case}.dur"].sum(1) * vc.hop).tolist()


@pytest.mark.gpu
def test_without_predictor_dur_prediction_still_raises():
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    voc = load_vocoder_model("tiny", synthetic=True)
    assert not voc.code_generator.has_dur_predictor
    with pytest.raises(NotImplementedError):
        voc(torch.zeros(1, 4, dtype=torch.int64, device=dev), "spa", -1)


@pytest.mark.gpu
def test_full_width_matches_oracle():
    """base arch (predictor 1280 -> 1280, k3): durations against the fp32 oracle, allowing a flip only where the oracle's
    exp(l) - 1 lies within 0.02 of a half-integer; waveforms of a ragged batch against the oracle given the same
    durations."""
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    vc = C.base_vocoder()
    vsd = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
    eng = load_vocoder_model("vocoder_v2", state_dict=vsd).code_generator
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    g = torch.Generator().manual_seed(5)
    units = torch.randint(0, vc.num_embeddings, (4, 48), generator=g)
    lang, spkr = [25, 8, 3, 30], [45, 10, 3, 120]
    _, raw, ref_dur = oracle_resynth(vc, vsd, units, lang, spkr)
    _, _, dur = eng.resynthesize(units.to(dev), lang, spkr)
    dur = dur.cpu().long()
    flips = (dur != ref_dur)
    near = ((raw - raw.floor()) - 0.5).abs() < 0.02
    assert not bool((flips & ~near).any()), f"{int(flips.sum())} durations differ, not all at rounding near-ties"
    assert ref_dur.min() == 1 and ref_dur.max() >= 4 and 1.5 < ref_dur.float().mean() < 3.0
    # waveform on a short ragged batch (the oracle's CPU HiFi-GAN at full width is slow on long rows)
    short = units[:, :10]
    d_short = ref_dur[:, :10].clone()
    d_short[1, 0] += 1  # totals differ
    ref_wav, _, _ = oracle_resynth(vc, vsd, short, lang, spkr, durations=d_short)
    wav, wav_lens, _ = eng.resynthesize(short.to(dev), lang, spkr, durations=d_short)
    assert wav_lens.tolist() == (d_short.sum(1) * vc.hop).tolist()
    assert wav.shape == ref_wav.shape
    err = (wav.cpu() - ref_wav).abs().max().item()
    assert err < 5e-3, err
    for b in range(4):
        assert not wav[b, 0, int(wav_lens[b]):].any()


@pytest.mark.gpu
def test_zero_projection_gives_unit_durations_and_the_plain_path(tiny):
    """proj weight 0, bias 0: exp(0) - 1 = 0 rounds to 0, clamped to 1, so every unit lasts one frame and the
    waveform equals dur_prediction=False bit for bit."""
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    vc, vsd, _ = tiny
    sd = dict(vsd)
    sd[f"{P}.dur_predictor.proj.weight"] = torch.zeros_like(sd[f"{P}.dur_predictor.proj.weight"])
    sd[f"{P}.dur_predictor.proj.bias"] = torch.zeros(1)
    voc = load_vocoder_model("tiny", state_dict=sd)
    eng = voc.code_generator
    units = torch.randint(0, vc.num_embeddings, (3, 29), generator=torch.Generator().manual_seed(2)).to(dev)
    for _ in _both_resblock_paths(eng):
        a = voc(units, "spa", -1, dur_prediction=True)
        b = voc(units, "spa", -1, dur_prediction=False)
        assert voc.last_wav_lens.tolist() == [29 * vc.hop] * 3
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_equal_totals_equal_host_expanded_units(tiny):
    """Rows with equal totals: the device expansion + masked generator equals the plain generator on units expanded
    with repeat_interleave on the host, bit for bit (predicted durations, and overridden ones)."""
    vc, _, voc = tiny
    eng = voc.code_generator
    g = torch.Generator().manual_seed(4)
    row = torch.randint(0, vc.num_embeddings, (1, 21), generator=g)
    d = np.load(os.path.join(G, "codehifigan_dur_tiny.npz"))
    over = torch.tensor([[1, 2, 3, 4, 5, 6], [6, 5, 4, 3, 2, 1], [3, 4, 4, 3, 4, 3]])
    cases = [(row.repeat(3, 1), None), (torch.from_numpy(d["two.units"]), None),
             (torch.randint(0, vc.num_embeddings, (3, 6), generator=g), over)]
    for _ in _both_resblock_paths(eng):
        for units, dur_in in cases:
            B = units.shape[0]
            lang, spkr = [25, 8, 3][:B], [45, 10, 3][:B]
            wav, _, dur = eng.resynthesize(units.to(dev), lang, spkr, durations=dur_in)
            dur = dur.cpu().long()
            assert len(set(dur.sum(1).tolist())) == 1
            expanded = torch.stack([units[b].repeat_interleave(dur[b]) for b in range(B)])
            assert torch.equal(wav, eng(expanded.to(dev), lang, spkr))


def _ragged_cases(vc):
    g = torch.Generator().manual_seed(6)
    r = lambda shape: torch.randint(0, vc.num_embeddings, shape, generator=g)
    long_dur = torch.randint(30, 51, (3, 6), generator=g)  # rows end mid-tile at different places, several tiles each
    return [
        ("U=1", r((3, 1)), torch.tensor([[1], [2], [5]])),
        ("long", r((3, 6)), long_dur),
        ("off-by-one", r((3, 3)), torch.tensor([[3, 4, 5], [3, 4, 6], [3, 4, 4]])),
        ("predicted", r((4, 13)), None),
    ]


@pytest.mark.gpu
def test_ragged_rows_equal_rows_vocoded_alone(tiny):
    """Row b of a ragged batch: its first hop*T_b samples equal that row vocoded alone bit for bit, the rest are 0;
    on the fused ResBlock kernel and conv by conv."""
    vc, _, voc = tiny
    eng = voc.code_generator
    for fused in _both_resblock_paths(eng):
        for name, units, dur_in in _ragged_cases(vc):
            B = units.shape[0]
            lang, spkr = [25, 8, 3, 30][:B], [45, 10, 3, 120][:B]
            wav, wav_lens, dur = eng.resynthesize(units.to(dev), lang, spkr, durations=dur_in)
            dur = dur.cpu()
            assert wav_lens.tolist() == (dur.long().sum(1) * vc.hop).tolist()
            assert wav.shape == (B, 1, int(wav_lens.max()))
            if name != "predicted":
                assert len(set(wav_lens.tolist())) == B, name  # really ragged
            for b in range(B):
                n = int(wav_lens[b])
                alone, _, _ = eng.resynthesize(units[b:b + 1].to(dev), lang[b:b + 1], spkr[b:b + 1], durations=dur[b:b + 1])
                assert alone.shape == (1, 1, n)
                assert torch.equal(wav[b, :, :n], alone[0]), (fused, name, b, float((wav[b, :, :n] - alone[0]).abs().max()))
                assert not wav[b, :, n:].any(), (fused, name, b)


@pytest.mark.gpu
def test_repeated_calls_are_bit_identical(tiny):
    vc, _, voc = tiny
    units = torch.randint(0, vc.num_embeddings, (4, 31), generator=torch.Generator().manual_seed(9)).to(dev)
    a = voc(units, ["spa", "eng", "deu", "fra"], -1)
    la = voc.last_wav_lens.clone()
    b = voc(units, ["spa", "eng", "deu", "fra"], -1)
    assert torch.equal(a, b) and torch.equal(la, voc.last_wav_lens)
