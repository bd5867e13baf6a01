"""seamlessM4T_large (w2v-BERT v1 speech encoder): Transformer-XL relative attention (`sb_attention_relpos`), the
symmetric depthwise conv with folded BatchNorm (`sb_dwconv_bias_silu`), the v1 engine path, loading and S2TT / ASR.

CPU tests pin the v1 oracle (tests/oracle_v1.py) to `UnityOracle`'s mirror-pinned v1 block and the recalled position
table; GPU tests hold the kernels to float64 / fp32 references and the engine to the oracle."""
import dataclasses
import hashlib
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle.unity_oracle import fbank as o_fbank
from oracle_v1 import N_CTX, UnityOracleV1, relpos_index, relpos_table, shift_bd
from seamless_communication_b200 import config as C, synthetic as S
from seamless_communication_b200.models import checkpoint as ck

dev = "cuda"
gpu = pytest.mark.gpu


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-9)).item()


# ------------------------------------------------------------------------------------------------ fairseq names
_LAYER = [("ffn1_layer_norm.", "ffn1.layer_norm."), ("ffn2_layer_norm.", "ffn2.layer_norm."), ("ffn1.inner_proj.", "ffn1.w_1."),
          ("ffn1.output_proj.", "ffn1.w_2."), ("ffn2.inner_proj.", "ffn2.w_1."), ("ffn2.output_proj.", "ffn2.w_2."),
          ("self_attn_layer_norm.", "self_attn_layer_norm."), ("self_attn.q_proj.", "self_attn.linear_q."),
          ("self_attn.k_proj.", "self_attn.linear_k."), ("self_attn.v_proj.", "self_attn.linear_v."),
          ("self_attn.output_proj.", "self_attn.linear_out."), ("self_attn.sdpa.r_proj.", "self_attn.linear_pos."),
          ("self_attn.sdpa.u_bias", "self_attn.pos_bias_u"), ("self_attn.sdpa.v_bias", "self_attn.pos_bias_v"),
          ("conv_layer_norm.", "conv_module.layer_norm."), ("conv.", "conv_module."), ("layer_norm.", "final_layer_norm.")]
_ADAPTOR = [("residual_conv.", "residual_pool.1."), ("self_attn_conv.", "attn_pool.1."), ("self_attn.output_proj.", "self_attn.out_proj."),
            ("ffn.inner_proj.", "fc1."), ("ffn.output_proj.", "fc2."), ("ffn_layer_norm.", "final_layer_norm."), ("", "")]
_DEC = [("self_attn.output_proj.", "self_attn.out_proj."), ("encoder_decoder_attn.output_proj.", "encoder_attn.out_proj."),
        ("encoder_decoder_attn_layer_norm.", "encoder_attn_layer_norm."), ("encoder_decoder_attn.", "encoder_attn."),
        ("ffn.inner_proj.", "fc1."), ("ffn.output_proj.", "fc2."), ("ffn_layer_norm.", "final_layer_norm."), ("", "")]
W2V = "encoder.w2v_encoder.w2v_model."


def _sub(rest, table):
    for a, b in table:
        if rest.startswith(a):
            return b + rest[len(a):]
    raise KeyError(rest)


def to_fairseq(key: str) -> str:
    """fairseq2 name of a v1 synthetic parameter -> the original fairseq name (inverse of checkpoint.rename_key)."""
    fixed = {"speech_encoder.inner_layer_norm.": W2V + "encoder.layer_norm.", "speech_encoder.proj1.": "encoder.adaptor.proj.0.",
             "speech_encoder.proj2.": "encoder.adaptor.proj.2.", "speech_encoder.layer_norm.": "encoder.adaptor.out_ln.",
             "speech_encoder_frontend.post_extract_layer_norm.": W2V + "layer_norm.",
             "speech_encoder_frontend.model_dim_proj.": W2V + "post_extract_proj.",
             "text_decoder_frontend.embed.": "target_letter_decoder.embed_tokens.", "final_proj.": "target_letter_decoder.output_projection.",
             "text_decoder.layer_norm.": "target_letter_decoder.layer_norm."}
    for a, b in fixed.items():
        if key.startswith(a):
            return b + key[len(a):]
    parts = key.split(".")
    if key.startswith("speech_encoder.inner.layers."):
        return f"{W2V}encoder.layers.{parts[3]}." + _sub(".".join(parts[4:]), _LAYER)
    if key.startswith("speech_encoder.adaptor_layers."):
        return f"encoder.adaptor.layers.{parts[2]}." + _sub(".".join(parts[3:]), _ADAPTOR)
    if key.startswith("text_decoder.layers."):
        return f"target_letter_decoder.layers.{parts[2]}." + _sub(".".join(parts[3:]), _DEC)
    raise KeyError(key)


def fairseq_checkpoint(sd):
    """A fairseq-named checkpoint that convert_unity_checkpoint turns back into `sd` (control rows pre-permuted), plus
    an AR T2U and a text encoder parameter that loading a v1 model must drop."""
    fs = {to_fairseq(k): v.clone() for k, v in sd.items() if k != "text_decoder_frontend.embed.weight"}
    emb = sd["final_proj.weight"].clone()
    emb[[1, 3, 0, 2]] = sd["final_proj.weight"][[0, 1, 2, 3]]
    fs["target_letter_decoder.output_projection.weight"] = emb
    fs["decoder.layers.0.self_attn.k_proj.weight"] = torch.zeros(4, 4)
    fs["synthesizer_encoder.layers.0.fc1.weight"] = torch.zeros(4, 4)
    fs["text_encoder.layers.0.fc1.weight"] = torch.zeros(4, 4)
    return {"model": fs}


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("S", [1, 2, 7, 64, 65])
def test_relative_shift_closed_form(S):
    """The index S-1+j-i reproduces the oracle's pad / reshape / slice shift exactly, and the masked batched attention
    built on it equals the oracle's own unpadded `mha_relpos_v1`."""
    bd = torch.arange(2 * 3 * S * (2 * S - 1), dtype=torch.float64).view(2, 3, S, 2 * S - 1)
    assert torch.equal(shift_bd(bd), torch.gather(bd, 3, relpos_index(S).expand(2, 3, S, S)))
    cfg = C.tiny_v1()
    sd = S_v1_tiny()
    uo = UnityOracleV1(cfg.to_dict(), sd)
    x = torch.randn(1, S, cfg.model_dim, generator=torch.Generator().manual_seed(S))
    p = "speech_encoder.inner.layers.0.self_attn"
    assert (uo.mha_relpos(p, x) - uo.mha_relpos_v1(p, x, uo.pos_enc)).abs().max() < 1e-5


def S_v1_tiny(seed=0):
    return S.make_unity_state_dict(C.tiny_v1(), seed, dec_gain=4.0)


def test_relpos_table_recalled_formula():
    from seamless_communication_b200.engine import XL_POS_CTX, relpos_table as eng_table
    M = 64
    t = relpos_table(N_CTX, M)
    assert XL_POS_CTX == N_CTX and t.shape == (2 * N_CTX - 1, M)
    assert torch.equal(t[N_CTX - 1], torch.tensor([0.0, 1.0] * (M // 2)))   # step 0
    s = torch.arange(1, N_CTX)
    assert torch.equal(t[N_CTX - 1 - s][:, 0::2], -t[N_CTX - 1 + s][:, 0::2])  # sin: odd in the step
    assert torch.equal(t[N_CTX - 1 - s][:, 1::2], t[N_CTX - 1 + s][:, 1::2])   # cos: even in the step
    assert abs(float(t[N_CTX - 2, 0]) - math.sin(1.0)) < 1e-7                    # row n_ctx-2 holds step +1
    assert (eng_table(N_CTX, M) - t).abs().max() < 1e-6                          # the engine's table is the same formula
    # a state dict's speech_encoder.pos_enc replaces the formula
    cfg = C.tiny_v1()
    sd = S_v1_tiny()
    pe = torch.randn(2 * N_CTX - 1, cfg.model_dim, generator=torch.Generator().manual_seed(3))
    x = torch.randn(2, 9, cfg.model_dim, generator=torch.Generator().manual_seed(4))
    p = "speech_encoder.inner.layers.0.self_attn"
    a = UnityOracleV1(cfg.to_dict(), sd).mha_relpos(p, x)
    b = UnityOracleV1(cfg.to_dict(), {**sd, "speech_encoder.pos_enc": pe}).mha_relpos(p, x)
    assert torch.equal(UnityOracleV1(cfg.to_dict(), {**sd, "speech_encoder.pos_enc": pe}).pos_enc, pe)
    assert (a - b).abs().max() > 1e-2


def test_masked_oracle_rows_equal_rows_alone():
    """Each valid row of a ragged batch equals that row encoded alone (Conformer stack output, within 1e-5)."""
    cfg = C.tiny_v1()
    uo = UnityOracleV1(cfg.to_dict(), S_v1_tiny())
    g = torch.Generator().manual_seed(5)
    fb = torch.randn(3, 90, 80, generator=g)
    lens = torch.tensor([90, 61, 2])
    for i in range(3):
        fb[i, lens[i]:] = 0
    _, _, inner = uo.encode_speech(fb, lens, return_inner=True)
    for i in range(3):
        n = int(lens[i])
        _, _, alone = uo.encode_speech(fb[i:i + 1, :n], None, return_inner=True)
        assert (inner[i, :n // 2] - alone[0]).abs().max() < 1e-5


def test_v1_config_and_state_dict():
    assert C.MODEL_CARDS["seamlessM4T_large"] == "base"
    b, b2 = C.base(), C.base_v2()
    assert b.encoder_variant == "v1" and b2.encoder_variant == "v2"
    assert dataclasses.replace(b, name=b2.name, encoder_variant="v2") == b2
    for arch in ("tiny_v1", "small_v1"):
        c = C.UNITY_ARCHS[arch]()
        assert c.encoder_variant == "v1"
    sd = S_v1_tiny()
    cfg = C.tiny_v1()
    p = "speech_encoder.inner.layers.1"
    assert sd[p + ".self_attn.sdpa.u_bias"].shape == (cfg.num_heads, 64) and sd[p + ".self_attn.sdpa.v_bias"].shape == (cfg.num_heads, 64)
    assert sd[p + ".self_attn.sdpa.r_proj.weight"].shape == (cfg.model_dim, cfg.model_dim)
    assert p + ".self_attn.sdpa.r_proj.bias" not in sd
    rv, rm = sd[p + ".conv.batch_norm.running_var"], sd[p + ".conv.batch_norm.running_mean"]
    assert rv.min() > 0.2 and rv.std() > 0.2 and rm.abs().max() > 0.2
    assert not any("rel_k_embed" in k or k.startswith("t2u_model.") or "conv.layer_norm." in k for k in sd)


# sha256 over sorted (name, tensor bytes) of the v2 synthetic state dicts, as drawn before the v1 variant existed
V2_HASHES = {("tiny_v2", 0): "5e9f4e7a6ab9ed52dd27eba1418625df0dc3e5ef2543c66567b9bae1337de9c5",
             ("tiny_v2", 7): "50ebe4ddc2a1f02a9c79cc5a6799443e0a989243f4f4e8c7979025b9eac5c97a",
             ("small_v2", 0): "163b3b011d207225d631b39b4daa37a1d6442b75bf2dacac9c793083eb8543df",
             ("small_v2", 7): "e0a39f85df0dd934d364a4d01ec6923829f46d3c2511f1970a4d6d8f1d43ce0f"}


def test_v2_state_dicts_unchanged():
    for (arch, seed), want in V2_HASHES.items():
        sd = S.make_unity_state_dict(C.UNITY_ARCHS[arch](), seed)
        h = hashlib.sha256()
        for k in sorted(sd):
            h.update(k.encode())
            h.update(sd[k].contiguous().numpy().tobytes())
        assert h.hexdigest() == want, (arch, seed)


def test_v1_fairseq_names_convert():
    sd = S_v1_tiny()
    for k in sd:
        if k != "text_decoder_frontend.embed.weight":
            assert ck.rename_key(to_fairseq(k)) == k, (k, to_fairseq(k))
    fs = fairseq_checkpoint(sd)
    fs["model"] = {k: v for k, v in fs["model"].items() if not k.startswith(("decoder.", "synthesizer_encoder.", "text_encoder."))}
    out = ck.convert_unity_checkpoint(fs, nllb_vocab=C.tiny_v1().text_vocab)["model"]
    assert sorted(out) == sorted(sd)
    for k in sd:
        assert torch.equal(out[k], sd[k]), k


# ------------------------------------------------------------------------------------------------ GPU: kernels
def _attn_ref64(q, k, v, r, u, vb, lens, S, H):
    """float64 reference from the kernel's own fp16 inputs: q + u and q + v summed in fp32 and rounded to fp16 once."""
    B = q.shape[0]
    out = torch.zeros(B, S, H * 64, dtype=torch.float64, device=q.device)
    idx = relpos_index(S).to(q.device)
    for b in range(B):
        L = int(lens[b])
        for h in range(H):
            sl = slice(64 * h, 64 * h + 64)
            qh = q[b, :, sl].float()
            qu = (qh + u[h]).half().double()
            qv = (qh + vb[h]).half().double()
            kk, vv = k[b, :L, sl].double(), v[b, :L, sl].double()
            bd = qv @ r[:, sl].double().t()                          # (S, 2S-1)
            s = (qu @ kk.t() + torch.gather(bd, 1, idx[:, :L])) / 8
            out[b, :, sl] = torch.softmax(s, dim=1) @ vv
    return out


def _relpos_case(ops, S, H, B, seed, lens=None):
    g = torch.Generator(device=dev).manual_seed(seed)
    M = 64 * H
    if lens is None:
        lens = torch.full((B,), S, dtype=torch.int32)
        if B > 1:
            lens[1] = 1
        for b in range(2, B):
            lens[b] = max(1, S - 37 * b)
    lens_d = lens.to(dev, torch.int32)
    qkv = torch.randn(B, S, 3 * M, device=dev, generator=g).half()
    for b in range(B):  # key / value rows past the length hold NaN: a stray read poisons the output
        qkv[b, int(lens[b]):, M:] = float("nan")
    r = (torch.randn(2 * S - 1, M, device=dev, generator=g)).half()
    u = torch.randn(H, 64, device=dev, generator=g) * 0.5
    vb = torch.randn(H, 64, device=dev, generator=g) * 0.5
    buf = qkv.view(B * S, 3 * M)
    out = torch.full((B * S, M), float("nan"), device=dev, dtype=torch.float16)
    ops.attention_relpos(buf[:, :M], buf[:, M:2 * M], buf[:, 2 * M:], out, B, H, S, S, 0, S, 0, r, u, vb, lens_d)
    return qkv, r, u, vb, lens, out.view(B, S, M)


@gpu
@pytest.mark.parametrize("H", [2, 16])
@pytest.mark.parametrize("S", [1, 2, 63, 64, 65, 127, 128, 129, 499, 500, 1000, 4096])
def test_attention_relpos_matches_float64(S, H):
    """Bound |out - ref| <= 2^-11 |ref| + 2^-11 max|v| + 1e-5: the output is rounded to fp16 (2^-11 relative) and the
    kernel multiplies V by exp(s - m) rounded to fp16 (relative error <= 2^-11 for every weight) while normalising by
    the fp32 sum, which moves the output by at most 2^-11 sum_j p_j |v_j| / l <= 2^-11 max|v|.  That is looser than
    test_decode_attention's 2e-4 max|v|, whose kernels keep the weights in fp32.  Score arithmetic is fp32 over 64
    terms (relative error ~1e-6) and is covered by the 1e-5 term."""
    from seamless_communication_b200 import ops
    B = 1 + S % 5
    M = 64 * H
    qkv, r, u, vb, lens, out = _relpos_case(ops, S, H, B, seed=S * 31 + H)
    ref = _attn_ref64(qkv[..., :M], qkv[..., M:2 * M], qkv[..., 2 * M:], r, u, vb, lens, S, H)
    assert torch.isfinite(out).all()
    for b in range(B):
        vmax = qkv[b, :int(lens[b]), 2 * M:].float().abs().max().item()
        err = (out[b].double() - ref[b]).abs()
        bound = 2 ** -11 * ref[b].abs() + 2 ** -11 * vmax + 1e-5
        assert (err <= bound).all(), (b, (err - bound).max().item())
    # without u / v the kernel computes q.k + q.R
    buf = qkv.view(B * S, 3 * M)
    out0 = torch.empty(B * S, M, device=dev, dtype=torch.float16)
    ops.attention_relpos(buf[:, :M], buf[:, M:2 * M], buf[:, 2 * M:], out0, B, H, S, S, 0, S, 0, r, None, None, lens.to(dev))
    z = torch.zeros(H, 64, device=dev)
    ref0 = _attn_ref64(qkv[..., :M], qkv[..., M:2 * M], qkv[..., 2 * M:], r, z, z, lens, S, H)
    assert ((out0.view(B, S, M).double() - ref0).abs() <= 2 ** -11 * ref0.abs() + 2 ** -11 * qkv[..., 2 * M:].nan_to_num(0).float().abs().max() + 1e-5).all()


@gpu
def test_attention_relpos_rows_independent_and_limits():
    """A row's output does not depend on the other rows of the batch (bit for bit), repeated calls are bit-identical,
    and S > 4096 returns SB_ENOSUP without launching anything."""
    from seamless_communication_b200 import _lib, ops
    S, H, B = 300, 16, 3
    lens = torch.tensor([300, 211, 1], dtype=torch.int32)
    qkv, r, u, vb, _, out = _relpos_case(ops, S, H, B, seed=11, lens=lens)
    M = 64 * H
    _, _, _, _, _, again = _relpos_case(ops, S, H, B, seed=11, lens=lens)
    assert torch.equal(out, again)
    one = torch.empty(S, M, device=dev, dtype=torch.float16)
    b1 = qkv[1].contiguous()
    ops.attention_relpos(b1[:, :M], b1[:, M:2 * M], b1[:, 2 * M:], one, 1, H, S, S, 0, S, 0, r, u, vb, lens[1:2].to(dev))
    assert torch.equal(one, out[1])
    lib = _lib.load()
    S2 = 4097
    x = torch.zeros(S2, 3 * 128, device=dev, dtype=torch.float16)
    r2 = torch.zeros(2 * S2 - 1, 128, device=dev, dtype=torch.float16)
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    rc = lib.sb_attention_relpos(x.data_ptr(), x.stride(0), x[:, 128:].data_ptr(), x.stride(0), x[:, 256:].data_ptr(), x.stride(0),
                                 x.data_ptr(), x.stride(0), 1, 2, S2, S2, 0, S2, 0, None, r2.data_ptr(), 128, None, None,
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == -3 and lib.sb_launch_count() == n0


@gpu
@pytest.mark.parametrize("C_", [128, 1024])
def test_dwconv_bias_silu_matches_fp32(C_):
    """Symmetric k=31 depthwise conv + bias + SiLU against fp32 torch at T straddling the 32-frame tiles, with ragged rows
    zero past their ends (as the encoder leaves them): bound 2^-10 |ref| + 1e-4 (fp16 output rounding + fp32 sums)."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.ops import Seq
    g = torch.Generator(device=dev).manual_seed(C_)
    for T in (1, 15, 31, 32, 33, 47, 64, 95, 499):
        B = 3
        lens = [T, max(1, T - 17), 1]
        x = torch.randn(B, T, C_, device=dev, generator=g).half()
        for b in range(B):
            x[b, lens[b]:] = 0
        w = (torch.randn(C_, 31, device=dev, generator=g) / math.sqrt(31)).half()
        bias = torch.randn(C_, device=dev, generator=g) * 0.3
        y = ops.dwconv_bias_silu(Seq(B, T, C_, buf=x.view(B * T, C_)), w, bias, 31).buf.view(B, T, C_)
        ref = F.silu(F.conv1d(F.pad(x.float().transpose(1, 2), (15, 15)), w.float()[:, None], groups=C_) + bias[:, None]).transpose(1, 2)
        assert ((y.float() - ref).abs() <= 2 ** -10 * ref.abs() + 1e-4).all(), T
        for b in range(B):  # each row equals the row alone
            yb = ops.dwconv_bias_silu(Seq(1, lens[b], C_, buf=x[b, :lens[b]].contiguous()), w, bias, 31).buf
            assert torch.equal(yb, y[b, :lens[b]])


# ------------------------------------------------------------------------------------------------ GPU: engine
@pytest.fixture(scope="module")
def tiny1():
    from seamless_communication_b200.models.unity import load_unity_model
    cfg = C.tiny_v1()
    sd = S_v1_tiny()
    toks = S.make_tokenizers(cfg)
    model = load_unity_model("tiny_v1", state_dict=sd, tokenizers=toks)
    return dict(cfg=cfg, sd=sd, toks=toks, model=model, uo=UnityOracleV1(cfg.to_dict(), sd, toks))


def _ragged_fbank(ops):
    waves = S.make_waveforms(3, 32000)
    ns = torch.tensor([32000, 23456, 16001], dtype=torch.int32)
    fb, frames = ops.fbank(waves.to(dev), ns.to(dev), 198)
    ofb = torch.zeros(3, 198, 80)
    for i in range(3):
        f = o_fbank(waves[i, :ns[i]])
        ofb[i, :f.shape[0]] = f
    return fb, frames, ofb


@gpu
def test_encoder_tiny_v1_matches_oracle_ragged(tiny1):
    from seamless_communication_b200 import ops
    fb, frames, ofb = _ragged_fbank(ops)
    eng, uo = tiny1["model"].engine, tiny1["uo"]
    enc, lens, inner = eng.encode_speech(fb, frames, return_inner=True)
    o_enc, o_lens, o_inner = uo.encode_speech(ofb, frames.cpu().long(), return_inner=True)
    assert lens.tolist() == o_lens.tolist()
    M = tiny1["cfg"].model_dim
    for i in range(3):
        n_in, n_out = int(frames[i]) // 2, int(o_lens[i])
        assert rel(inner.buf.view(3, -1, M)[i, :n_in], o_inner[i, :n_in]) < 5e-3
        assert rel(enc.buf.view(3, -1, M)[i, :n_out], o_enc[i, :n_out]) < 5e-3


@gpu
def test_encoder_base_full_width_matches_oracle():
    """`base` encoder at full width (24 layers, 1024 dims, 16 heads) on one 10 s utterance against the fp32 oracle, run
    on the GPU in fp32 (TF32 off).  Only the encoder is compared, so the text decoder is cut to one layer and a small
    vocabulary to keep the synthetic state dict small."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.engine import UnitYEngine
    cfg = dataclasses.replace(C.base(), dec_layers=1, text_vocab=8192 + 102)
    sd = S.make_unity_state_dict(cfg, 3)
    eng = UnitYEngine(cfg, sd, S.make_tokenizers(cfg))
    wave = S.make_waveforms(1, 160000, seed=21)
    fb, frames = ops.fbank(wave.to(dev), torch.tensor([160000], dtype=torch.int32, device=dev), 998)
    enc, _ = eng.encode_speech(fb, None)
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        uo = UnityOracleV1(cfg.to_dict(), {k: v.to(dev) for k, v in sd.items() if not k.startswith(("text_", "final_"))})
        o_enc, _ = uo.encode_speech(o_fbank(wave[0]).to(dev)[None, :998], None)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    err = rel(enc.buf.view(1, -1, 1024)[0], o_enc[0])
    print(f"base v1 encoder rel err {err:.2e}")
    assert err < 5e-3


@gpu
def test_small_v1_rows_independent_and_deterministic():
    """Permuting a ragged small_v1 batch permutes the output bit for bit and repeated calls are bit-identical.  A row
    encoded alone agrees with its batched frames to 2e-3, not bit for bit: the GEMM picks its tile shape from the row
    count (the v2 path has the same exception, test_full_width_properties_permutation_padding_determinism)."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.models.unity import load_unity_model
    eng = load_unity_model("small_v1", synthetic=True, seed=7, dec_gain=4.0).engine
    waves = S.make_waveforms(4, 160000, seed=9)
    ns = torch.tensor([160000, 101234, 96000, 40000], dtype=torch.int32)
    fb, frames = ops.fbank(waves.to(dev), ns.to(dev), 998)
    enc, lens, inner = eng.encode_speech(fb, frames, return_inner=True)
    M = 1024
    e, ei = enc.buf.view(4, -1, M).clone(), inner.buf.view(4, -1, M).clone()
    enc2, _ = eng.encode_speech(fb, frames)
    assert torch.equal(e, enc2.buf.view(4, -1, M))
    perm = [2, 0, 3, 1]
    encp, _, innerp = eng.encode_speech(fb[perm].contiguous(), frames[perm].contiguous(), return_inner=True)
    assert torch.equal(innerp.buf.view(4, -1, M), ei[perm]) and torch.equal(encp.buf.view(4, -1, M), e[perm])
    for i in (1, 3):
        n = int(frames[i])
        _, _, alone = eng.encode_speech(fb[i:i + 1, :n + (n % 2)].contiguous(), frames[i:i + 1].contiguous(), return_inner=True)
        assert rel(alone.buf.view(1, -1, M)[0, :n // 2], ei[i, :n // 2]) < 2e-3
    assert torch.isfinite(e).all() and e.float().std() > 0.1
    with pytest.raises(ValueError, match="maximum sequence length"):
        eng.encode_speech(torch.zeros(1, 2 * 4097, 80, dtype=torch.float16, device=dev), None)


@gpu
def test_translator_s2tt_asr_match_oracle(tiny1):
    """S2TT and ASR through Translator.predict on tiny_v1: the hypotheses equal the oracle's or differ only as a near tie
    under the oracle's own scoring (ASSUMPTIONS.md #9).  S2ST and T2ST raise NotImplementedError naming the AR T2U."""
    from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator
    model, uo, toks = tiny1["model"], tiny1["uo"], tiny1["toks"]
    tr = Translator(model, None, device="cuda:0")
    waves = S.make_waveforms(2, 32000, seed=77)
    opts = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=20)
    fb = torch.stack([o_fbank(w) for w in waves])
    for task, lang in (("s2tt", "spa"), ("asr", "eng")):
        texts, speech = tr.predict(tr.fbank_batch(waves), task, lang, text_generation_opts=opts)
        assert speech is None and len(texts) == 2
        ref = uo.generate(fb, None, lang, hard_max=20, output_units=False)
        hyps = Translator._last_generator.last_text_output.hypotheses
        for i in range(2):
            if hyps[i][0][1] != ref["text_ids"][i]:
                ids = torch.tensor(hyps[i][0][1])[None]
                h = uo.decoder(uo.embed_text(ids[:, :-1], 0), ref["enc"][i:i + 1], None)
                lp = torch.log_softmax(uo.project(h).float(), -1)[0]
                sc = sum(float(lp[t, ids[0, t + 1]]) for t in range(ids.shape[1] - 1)) / (ids.shape[1] - 1)
                assert abs(sc - ref["hyps"][i][0][0]) < 2e-2
            else:
                assert texts[i] == ref["texts"][i]
    for task in ("s2st", "t2st"):
        with pytest.raises(NotImplementedError, match="AR T2U"):
            tr.predict(tr.fbank_batch(waves), task, "spa", src_lang="eng")


@gpu
def test_fairseq_checkpoint_loads_same_encoder(tiny1):
    from seamless_communication_b200 import ops
    from seamless_communication_b200.models.unity import load_unity_model
    m2 = load_unity_model("tiny_v1", checkpoint=fairseq_checkpoint(tiny1["sd"]), tokenizers=tiny1["toks"])
    assert not m2.engine.has_t2u
    fb, frames, _ = _ragged_fbank(ops)
    a, la = tiny1["model"].engine.encode_speech(fb, frames)
    b, lb = m2.engine.encode_speech(fb, frames)
    assert torch.equal(a.buf, b.buf) and torch.equal(la, lb)
    assert torch.equal(m2.engine.w["text_embed"], tiny1["model"].engine.w["text_embed"])
