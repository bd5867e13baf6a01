"""XLS-R unit extractor (DESIGN.md section 11): the fp32 oracle against the reference's own code (fixture), the checkpoint
converter and the API's argument checks on the CPU; every new kernel against float64, the engine against the oracle,
ragged batches and the resynthesis hand-off on the GPU.

Tolerances of the kernel tests come from fp16 rounding: an fp16 store rounds to within 2^-11 relative (half an ulp of
the 11-bit significand), an fp16 operand of a tensor-core product carries the same relative error into each term, and
fp32 accumulation adds K * 2^-24 relative to the sum of |terms|, negligible next to the former at the K used here."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_w2v2 as O  # noqa: E402
from seamless_communication_b200 import config as C  # noqa: E402
from seamless_communication_b200 import synthetic as S  # noqa: E402
from seamless_communication_b200.models.checkpoint import convert_wav2vec2_checkpoint  # noqa: E402
from seamless_communication_b200.models.unit_extractor import UnitExtractor  # noqa: E402

G = os.path.join(ROOT, "tests", "golden")
FX = json.load(open(os.path.join(G, "unit_extractor.json")))
U16 = 2.0 ** -11  # fp16 unit roundoff


# ------------------------------------------------------------------------------------------------------------ CPU
def test_config_fields_equal_the_reference_architecture():
    ref = FX["arch"]["encoder"]
    cfg = C.xlsr2_1b_v2().to_dict()
    shared = [k for k in cfg if k in ref]
    assert len(shared) >= 15
    for k in shared:
        v = cfg[k]
        v = [list(x) for x in v] if k == "feature_extractor_layer_descs" else v
        assert v == ref[k], k
    # the fields the extractor does not model are the ones that do not change inference
    assert ref["use_fbank"] is False and ref["layer_drop_p"] == 0.0 and ref["first_pass_dropout_p"] == 0.0


def test_test_configs_keep_the_kernel_shapes():
    for cfg in (C.tiny_xlsr(), C.small_xlsr()):
        assert cfg.head_dim == 80 and cfg.model_dim // cfg.num_pos_conv_groups == 80
        assert cfg.feature_extractor_layer_descs == C.xlsr2_1b_v2().feature_extractor_layer_descs


def _kmeans_inputs():
    k = FX["kmeans"]
    g = torch.Generator().manual_seed(k["seed"])
    K, D, N = k["K"], k["D"], k["N"]
    c = torch.randn(K, D, generator=g)
    c[200] = c[7]
    c[299] = c[50]
    x = torch.randn(N, D, generator=g)
    x[:8] = c[7] + 0.01 * torch.randn(8, D, generator=g)
    x[8:16] = c[50] + 0.01 * torch.randn(8, D, generator=g)
    x[16] = c[299]
    return x, c


def test_oracle_kmeans_equals_the_reference():
    x, c = _kmeans_inputs()
    assert O.kmeans(x, c).tolist() == FX["kmeans"]["units"]
    assert FX["kmeans"]["units"][16] == 50  # exact duplicate: the lowest index


def test_frontend_keys_equal_the_reference_key_map():
    for k, ref in FX["frontend_keys"].items():
        out = convert_wav2vec2_checkpoint({"model": {k: torch.zeros(1)}})["model"]
        assert list(out) == [ref], (k, list(out), ref)


def _golden_generator():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_unit_extractor", os.path.join(G, "make_golden_unit_extractor.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_oracle_encoder_layers_match_reference_cpp():
    """The oracle's encoder layer (head split, head_dim^-0.5 scale, pre-LN order) at head_dim 80, run with ReLU in place of
    GELU and followed by the final LayerNorm, against the C++ mirror's StandardTransformerEncoder_forward
    (w2v2_encoder_ref.npz).  2e-3 as for the T2U encoder pin: ggml evaluates exp through an fp16 table."""
    gen = _golden_generator()
    ref = np.load(os.path.join(G, "w2v2_encoder_ref.npz"))
    P, M, H = gen.MIRROR["prefix"], gen.MIRROR["model_dim"], gen.MIRROR["num_heads"]
    assert M // H == 80
    for seed, S in gen.MIRROR_CASES:
        sd = gen.mirror_encoder_state_dict(seed)
        x = torch.from_numpy(ref[f"x_{seed}"])
        assert torch.equal(x, gen.mirror_input(seed, S))
        h = x
        for i in range(gen.MIRROR["layers"]):
            h = O.encoder_layer(h, S, sd, f"{P}.layers.{i}", H, act=F.relu)
        h = F.layer_norm(h, (M,), sd[P + ".layer_norm.weight"], sd[P + ".layer_norm.bias"], 1e-5)
        y = torch.from_numpy(ref[f"y_{seed}"])
        err = (h - y).abs().max().item()
        assert err < 2e-3, (seed, err)


def _fairseq_name(k: str) -> str:
    """fairseq2 name -> fairseq name (the inverse of convert_wav2vec2_checkpoint's rules)."""
    import re
    rules = [(r"^encoder_frontend\.pos_encoder\.conv\.", "encoder.pos_conv.0."),
             (r"^encoder_frontend\.feature_extractor\.layers\.(\d+)\.conv\.", r"feature_extractor.conv_layers.\1.0."),
             (r"^encoder_frontend\.feature_extractor\.layers\.(\d+)\.layer_norm\.", r"feature_extractor.conv_layers.\1.2.1."),
             (r"^encoder_frontend\.post_extract_layer_norm\.", "layer_norm."),
             (r"^encoder_frontend\.model_dim_proj\.", "post_extract_proj."),
             (r"\.self_attn\.output_proj\.", ".self_attn.out_proj."), (r"\.ffn\.inner_proj\.", ".fc1."),
             (r"\.ffn\.output_proj\.", ".fc2."), (r"\.ffn_layer_norm\.", ".final_layer_norm.")]
    for a, b in rules:
        k = re.sub(a, b, k)
    return k


def test_converter_round_trips_a_fairseq_named_dict():
    sd = S.make_wav2vec2_state_dict(C.tiny_xlsr(), seed=5)
    fs = {_fairseq_name(k): v for k, v in sd.items()}
    assert len(fs) == len(sd) and not any(k.startswith("encoder_frontend.") for k in fs)
    back = convert_wav2vec2_checkpoint({"model": fs})["model"]
    assert sorted(back) == sorted(sd)
    assert all(back[k] is sd[k] for k in sd)
    same = convert_wav2vec2_checkpoint({"model": sd})["model"]
    assert same == sd


def test_api_rejects_urls_wrong_widths_and_missing_weights(tmp_path):
    with pytest.raises(ValueError, match="URL"):
        UnitExtractor("tiny_xlsr", "https://example.org/kmeans_10k.npy", synthetic=True)
    p = str(tmp_path / "km.npy")
    np.save(p, np.zeros((16, 64), np.float32))
    with pytest.raises(ValueError, match="width"):
        UnitExtractor("tiny_xlsr", p, synthetic=True)
    np.save(p, np.zeros((16, 320), np.float32))
    with pytest.raises(RuntimeError, match="no weights"):
        UnitExtractor("tiny_xlsr", p)
    with pytest.raises(ValueError, match="unknown"):
        UnitExtractor("xlsr_nonexistent", p, synthetic=True)


def test_oracle_frame_counts():
    descs = C.xlsr2_1b_v2().feature_extractor_layer_descs
    assert O.conv_frames(160000, descs) == 499
    assert O.conv_frames(16079, descs) == 49 and O.conv_frames(16080, descs) == 50
    assert O.conv_frames(400, descs) == 1 and O.conv_frames(399, descs) == 0


# ------------------------------------------------------------------------------------------------------------ GPU
def _f64_front(wave, L, sd):
    x = wave[:L].double()
    if L % 2:
        x = torch.cat([x, torch.ones(1, dtype=torch.float64)])
    x = (x - x.mean()) / torch.sqrt(x.var(unbiased=False) + 1e-5)
    p = "encoder_frontend.feature_extractor.layers.0"
    h = F.conv1d(x.reshape(1, 1, -1), sd[p + ".conv.weight"].double(), sd[p + ".conv.bias"].double(), stride=5)[0].t()
    h = F.layer_norm(h, (512,), sd[p + ".layer_norm.weight"].double(), sd[p + ".layer_norm.bias"].double(), 1e-5)
    return F.gelu(h)


@pytest.mark.gpu
def test_front_kernel_against_float64():
    """Statistics + conv 0 + LayerNorm + GELU.  The kernel is fp32 throughout and rounds once to fp16, so each value is
    within 2^-11 |y| of the fp64 result plus the fp32 error of a 512-wide LayerNorm (~1e-5 |y| + 1e-6)."""
    from seamless_communication_b200 import ops
    sd = S.make_wav2vec2_state_dict(C.tiny_xlsr(), seed=7)
    lens = [400, 16079, 16000, 3201, 8000]
    B, Tm = len(lens), max(lens)
    g = torch.Generator().manual_seed(3)
    wave = torch.full((B, Tm + 16), float("nan"))
    for b, L in enumerate(lens):
        wave[b, :L] = 0.3 * torch.randn(L, generator=g) + 0.05
    rows = ((Tm + 1 - 10) // 5 + 1 + 63) // 64 * 64
    p = "encoder_frontend.feature_extractor.layers.0"
    out = ops.w2v2_front(wave.cuda(), torch.tensor(lens, dtype=torch.int32).cuda(),
                         sd[p + ".conv.weight"].reshape(512, 10).cuda(), sd[p + ".conv.bias"].cuda(),
                         sd[p + ".layer_norm.weight"].cuda(), sd[p + ".layer_norm.bias"].cuda(), rows)
    got = out.buf.view(B, rows, 512).double().cpu()
    for b, L in enumerate(lens):
        ref = _f64_front(wave[b], L, sd)
        T0 = ref.shape[0]
        assert torch.isfinite(got[b]).all()
        err = (got[b, :T0] - ref).abs()
        assert (err <= U16 * ref.abs() + 2e-5 * ref.abs().max() + 1e-6).all(), (L, err.max().item())
        assert (got[b, T0:] == 0).all()


@pytest.mark.gpu
def test_layernorm_gelu_against_float64():
    """fp16 input, fp32 statistics, one fp16 rounding of GELU(LN(x)): within 2^-11 |y| + 1e-4 max|y| (fp32 statistics of
    a 512-wide row and the erf evaluation)."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.ops import Seq
    B, T = 3, 300
    g = torch.Generator().manual_seed(4)
    x = (torch.randn(B * T, 512, generator=g) * 2 + 0.3).half()
    w = 1 + 0.1 * torch.randn(512, generator=g)
    bb = 0.1 * torch.randn(512, generator=g)
    lens = torch.tensor([300, 17, 150], dtype=torch.int32)
    y = ops.layernorm_gelu(Seq(B, T, 512, lens=lens.cuda(), buf=x.cuda()), w.cuda(), bb.cuda())
    ref = F.gelu(F.layer_norm(x.double(), (512,), w.double(), bb.double(), 1e-5)).view(B, T, 512)
    got = y.buf.view(B, T, 512).double().cpu()
    for b in range(B):
        n = int(lens[b])
        err = (got[b, :n] - ref[b, :n]).abs()
        assert (err <= U16 * ref[b, :n].abs() + 1e-4 * ref.abs().max()).all(), err.max().item()
        assert (got[b, n:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 16])
def test_attention_hd80_against_float64(heads):
    """Scores in fp32 from fp16 q, k; P rounded to fp16 before P.V (2^-11 relative per weight), output rounded to fp16:
    |err| <= 3 * 2^-11 * max|v| covers both roundings and the fp32 softmax.  Keys past kv_lens hold NaN (never read), rows
    past sq hold a sentinel (never written), kv_len 0 gives a zero row."""
    from seamless_communication_b200 import ops
    D = 80 * heads
    lens = [0, 1, 63, 64, 65, 1500] if heads == 1 else [1, 65, 640]
    B, T, pad = len(lens), max(lens) + 5, 2
    g = torch.Generator().manual_seed(heads)
    qkv = torch.randn(B, T + pad, 3 * D, generator=g).half()
    for b, n in enumerate(lens):
        qkv[b, n:, D:] = float("nan")
    out = torch.full((B * (T + pad), D), 7.0, dtype=torch.float16, device="cuda")
    buf = qkv.reshape(B * (T + pad), 3 * D).cuda()
    ops.attention_hd80(buf[:, :D], buf[:, D:2 * D], buf[:, 2 * D:], out, B, heads, T, T, T + pad, 0, T + pad, 0,
                       torch.tensor(lens, dtype=torch.int32).cuda())
    got = out.view(B, T + pad, D).double().cpu()
    for b, n in enumerate(lens):
        assert (got[b, T:] == 7.0).all()
        if n == 0:
            assert (got[b, :T] == 0).all()
            continue
        q, k, v = (qkv[b, :T, i * D:(i + 1) * D].double().view(T, heads, 80).transpose(0, 1) for i in range(3))
        k, v = k[:, :n], v[:, :n]
        ref = (torch.softmax(q @ k.transpose(1, 2) * 80 ** -0.5, -1) @ v).transpose(0, 1).reshape(T, D)
        err = (got[b, :T] - ref).abs().max().item()
        assert err <= 3 * U16 * v.abs().max().item(), (n, err)


@pytest.mark.gpu
def test_positional_conv_against_float64():
    """x + GELU(grouped conv) with the weight-norm fold: fp16 weights / inputs (2^-11 relative per product), fp32
    accumulation over 128 x 80 terms, one fp16 rounding: |err| <= 2^-11 (|y| + 2 sum|w||x|) per value."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.ops import Seq
    from seamless_communication_b200.wav2vec2_engine import Wav2Vec2Engine
    cfg = C.tiny_xlsr()
    sd = S.make_wav2vec2_state_dict(cfg, seed=9)
    eng = Wav2Vec2Engine(cfg, sd, S.make_kmeans_centroids(16, cfg.model_dim), device="cuda")
    M, lens = cfg.model_dim, [200, 37, 1]
    B, Te = len(lens), 200 + 64 + 8
    g = torch.Generator().manual_seed(5)
    x = torch.zeros(B, Te, M)
    for b, n in enumerate(lens):
        x[b, :n] = torch.randn(n, M, generator=g)
    x = x.half()
    out = Seq(B, Te, M, rows=Te, zero=False)
    ops.grouped_conv_gelu_res(Seq(B, Te, M, rows=Te, buf=x.reshape(B * Te, M).cuda()), eng.pos_w, eng.w["pos.b"], 128, out)
    got = out.buf.view(B, Te, M).double().cpu()
    w = O.pos_conv_weight({k: v.double() for k, v in sd.items()}).half().double()  # the fold, rounded like the packed weight
    # rows t < Te - 63 see only their own block (the zero rows after the previous block are their left padding); the
    # last 63 rows of a block read into the next one and carry no unit in the engine (Te >= frames + 64)
    R = Te - 63
    for b, n in enumerate(lens):
        xb = x[b].double()
        y = F.conv1d(xb.t()[None], w, sd["encoder_frontend.pos_encoder.conv.bias"].double(), padding=64, groups=4)[0, :, :-1].t()
        ref = xb + F.gelu(y)
        mag = F.conv1d(xb.abs().t()[None], w.abs(), None, padding=64, groups=4)[0, :, :-1].t()
        bound = U16 * (ref.abs() + 2 * mag) + 1e-6
        err = (got[b, :R] - ref[:R]).abs()
        assert (err <= bound[:R]).all(), (n, (err - bound[:R]).max().item())
    # the fold against weight_g * weight_v / ||weight_v|| computed independently per tap
    v, gg = sd["encoder_frontend.pos_encoder.conv.weight_v"].double(), sd["encoder_frontend.pos_encoder.conv.weight_g"].double()
    k = 17
    wk = gg[0, 0, k] * v[:, :, k] / v[:, :, k].norm()
    packed = eng.pos_w[1].double().cpu().view(80, 128, 80)[:, k]
    assert (packed - wk[80:160]).abs().max() <= U16 * wk.abs().max()


@pytest.mark.gpu
def test_nearest_centroid_full_width():
    """1280 x 10000 (a partial last tile of 16), exact duplicate centroids, rows past their length.  A differing unit is
    accepted only as a near-tie: the fp64 distance gap between the two centroids must lie within the fp32 accumulation
    bound 2 * 1280 * 2^-24 * sum|x||c| (x and c are already fp16)."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.ops import Seq
    K, D, B, T = 10000, 1280, 3, 130
    c = S.make_kmeans_centroids(K, D, seed=8, scale=0.05)
    c[9990] = c[3]
    c[9999] = c[128]
    g = torch.Generator().manual_seed(6)
    x = torch.randn(B * T, D, generator=g).half().float()
    x[0] = c[9990]
    x[1] = c[9999]
    lens = torch.tensor([130, 64, 1], dtype=torch.int32)
    x16 = x.half().cuda()
    nhn = (-0.5 * c.double().pow(2).sum(1)).float().cuda()
    units = ops.nearest_centroid(Seq(B, T, D, buf=x16), c.half().cuda(), nhn, lens.cuda()).view(B, T).cpu()
    dist = -2 * x.double() @ c.double().t() + c.double().pow(2).sum(1)[None]
    ref = dist.argmin(1).view(B, T)
    assert units[0, 0] == 3 and units[0, 1] == 128
    for b in range(B):
        n = int(lens[b])
        assert (units[b, n:] == -1).all()
        diff = (units[b, :n] != ref[b, :n]).nonzero().flatten()
        for t in diff.tolist():
            r = b * T + t
            gap = (dist[r, units[b, t]] - dist[r, ref[b, t]]).item()
            bound = 2 * D * 2.0 ** -24 * (x[r].abs() @ c.abs().t()).max().item() * 2
            assert 0 <= gap <= bound, (b, t, gap, bound)
        assert len(diff) <= max(1, n // 50)


def _waves(lens, seed=1):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(max(lens)) / 16000.0
    out = []
    for n in lens:
        f = 100 + 300 * torch.rand(1, generator=g).item()
        out.append((0.3 * torch.sin(2 * math.pi * f * t[:n]) + 0.05 * torch.randn(n, generator=g)).float())
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ["tiny_xlsr", "small_xlsr"])
def test_engine_against_the_oracle(arch):
    """Layer outputs at out_layer_idx in {0, middle, last} within 5e-3 of max|ref| (fp16 activations through the stack)."""
    cfg = C.WAV2VEC2_ARCHS[arch]()
    sd = S.make_wav2vec2_state_dict(cfg, seed=3)
    ue = UnitExtractor(arch, None, "cuda", state_dict=sd, synthetic=True, num_centroids=300)
    lens = [16079, 9000]
    waves = _waves(lens)
    batch = torch.zeros(len(lens), max(lens))
    for b, w in enumerate(waves):
        batch[b, :len(w)] = w
    L = cfg.num_encoder_layers
    for idx in (0, L // 2, L - 1):
        feats, n_out = ue.engine.forward(batch.cuda(), lens, idx)
        got = feats.buf.view(len(lens), feats.Tp, -1).float().cpu()
        for b, w in enumerate(waves):
            ref, _ = O.features(w, sd, cfg, idx)
            assert ref.shape[0] == n_out[b]
            err = (got[b, :n_out[b]] - ref).abs().max().item() / ref.abs().max().item()
            assert err < 5e-3, (arch, idx, b, err)


def _audit_units(units, ref_units, feats, ref_feats, centroids):
    """Every differing frame must be a near-tie: the oracle's fp64 distance gap between the two centroids is within what
    the frame's measured feature error e can move it: | |x+e-a|^2 - |x+e-b|^2 - (|x-a|^2 - |x-b|^2) | = 2 |e.(b-a)|."""
    diff = (units != ref_units).nonzero().flatten()
    for t in diff.tolist():
        a, b = int(units[t]), int(ref_units[t])
        gap = O.distance_gaps(ref_feats[t:t + 1], centroids, torch.tensor([a]), torch.tensor([b])).abs().item()
        e = (feats[t].double() - ref_feats[t].double()).norm().item()
        bound = 2 * e * (centroids[a].double() - centroids[b].double()).norm().item()
        assert gap <= bound, (t, gap, bound)
    return len(diff)


@pytest.mark.gpu
def test_full_width_xlsr2_1b_v2_layer_34():
    """xlsr2_1b_v2 at layer 34 on one 10 s utterance: features within 1e-2 of max|ref|, units equal up to near-ties."""
    cfg = C.xlsr2_1b_v2()
    sd = S.make_wav2vec2_state_dict(cfg, seed=3)
    ue = UnitExtractor("xlsr2_1b_v2", None, "cuda", state_dict=sd, synthetic=True)
    w = _waves([160000], seed=2)[0]
    feats, n_out = ue.engine.forward(w[None].cuda(), [160000], 34)
    units = ue.engine.units(feats, n_out)[0].cpu()
    got = feats.buf.float().cpu()[:n_out[0]]
    ref, _ = O.features(w, sd, cfg, 34)
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    print(f"xlsr2_1b_v2 layer 34: rel err {err:.2e}")
    assert err < 1e-2, err
    c = ue.engine.w["km.c"].float().cpu()
    ref_units = O.kmeans(ref, c)
    nd = _audit_units(units, ref_units, got, ref, c)
    print(f"units differing from the oracle: {nd} of {len(units)} (all near-ties)")


@pytest.mark.gpu
def test_predict_batch_ragged_rows_equal_predict_alone():
    lens = [16079, 400, 32000, 8000, 8001]
    ue = UnitExtractor("small_xlsr", None, "cuda", synthetic=True, num_centroids=500)
    waves = _waves(lens, seed=4)
    batch = torch.full((len(lens), max(lens) + 8), float("nan"))
    for b, w in enumerate(waves):
        batch[b, :len(w)] = w
    got = ue.predict_batch(batch.cuda(), lens, 3)
    descs = ue.cfg.feature_extractor_layer_descs
    for b, w in enumerate(waves):
        alone = ue.predict(w, 3)
        assert len(alone) == O.conv_frames(len(w) + len(w) % 2, descs)
        assert torch.equal(got[b], alone), b
    # the odd row of 16079 samples: 49 masked-valid frames, 50 units
    assert len(got[0]) == 50
    with pytest.raises(ValueError, match="400"):
        ue.predict(waves[0][:399], 3)
    with pytest.raises(ValueError, match="sampling rate"):
        ue.predict(waves[0], 3, sample_rate=8000)
    with pytest.raises(ValueError, match="out_layer_idx"):
        ue.predict(waves[0], 6)
    # a (T, 1) or (1, T) tensor is one channel; a multi-channel tensor is refused rather than collated differently
    assert torch.equal(ue.predict(waves[3][:, None], 3), got[3]) and torch.equal(ue.predict(waves[3][None], 3), got[3])
    with pytest.raises(ValueError, match="channel"):
        ue.predict(torch.stack([waves[3], waves[3]], 1), 3)
    with pytest.raises(ValueError, match="65535"):
        ue.engine.check_batch([160000] * 2000)


@pytest.mark.gpu
def test_predict_then_resynthesize_equals_the_vocoder(tmp_path):
    from seamless_communication_b200.evaluate import write_wav_f32
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    ue = UnitExtractor("tiny_xlsr", None, "cuda", synthetic=True, num_centroids=256)
    w = _waves([16079], seed=5)[0]
    p = str(tmp_path / "a.wav")
    write_wav_f32(p, w)
    units = ue.predict(p, 2)
    assert torch.equal(units, ue.predict(w, 2))
    vsd = S.make_vocoder_state_dict(C.tiny_vocoder(), 1, dur_predictor=True)
    wav = UnitExtractor.resynthesize_audio(units, "eng", "cuda", vocoder_name="vocoder_v2_tiny", state_dict=vsd)
    voc = load_vocoder_model("vocoder_v2_tiny", state_dict=vsd)
    direct = voc(units, "eng", -1, dur_prediction=True)
    assert torch.equal(wav, direct)
