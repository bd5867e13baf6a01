#!/usr/bin/env python
"""Staged bring-up checks on a real H100 (development aid; the tests live in tests/).
Usage: python tools/gpu_check.py [stage ...]   stages: gemm fbank ln attn dwconv encoder decode t2u vocoder e2e"""
import os
import sys
import time
import traceback

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.unity_oracle import UnityOracle, VocoderOracle, fbank as o_fbank, s2st  # noqa: E402
from seamless_communication_b200 import config as C, ops, synthetic as S  # noqa: E402
from seamless_communication_b200.ops import Seq  # noqa: E402

dev = "cuda"


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-9)).item()


def stage_gemm():
    torch.manual_seed(0)
    for (m, n, k) in [(128, 128, 64), (256, 128, 128), (300, 200, 1024), (160, 3072, 1024), (1000, 1024, 4096), (513, 72, 160)]:
        a = (torch.randn(m, k, device=dev) * 0.5).half()
        w = (torch.randn(n, k, device=dev) * 0.05).half()
        bias = torch.randn(n, device=dev)
        out = ops.gemm_raw(a, w, n, bias)
        ref = ops.gemm_raw(a, w, n, bias, ref=True)
        tref = a.float() @ w.float().t() + bias
        torch.cuda.synchronize()
        print(f"gemm {m}x{n}x{k}: tc-vs-simt {rel(out, ref):.2e}  tc-vs-torch {rel(out, tref):.2e}  simt-vs-torch {rel(ref, tref):.2e}")
    # conv taps + mask + residual + glu + dual output through the Seq interface
    B, T, Cc, N = 3, 50, 64, 96
    for taps, dil in [(3, 1), (7, 1), (11, 5), (1, 1)]:
        halo = (taps - 1) * dil // 2
        lens = torch.tensor([50, 33, 7], dtype=torch.int32, device=dev)
        x = Seq(B, T, Cc, halo=max(halo, 1), lens=lens)
        x.data().copy_((torch.randn(B, T, Cc, device=dev) * 0.5).half())
        w = (torch.randn(N, taps * Cc, device=dev) * 0.05).half()
        bias = torch.randn(N, device=dev)
        res = x.like(C=N, zero=True)
        res.data().copy_(torch.randn(B, T, N, device=dev).half())
        o2a, o2b = x.like(C=N, zero=True), x.like(C=N, zero=True)
        oa = ops.gemm(x, w, N, bias, taps=taps, dil=dil, act=ops.ACT_LRELU, slope=0.1, res1=res, alpha=0.5, out2=o2a, out2_slope=0.1)
        ob = ops.gemm(x, w, N, bias, taps=taps, dil=dil, act=ops.ACT_LRELU, slope=0.1, res1=res, alpha=0.5, out2=o2b, out2_slope=0.1, ref=True)
        # torch reference
        xc = x.data().float().transpose(1, 2)
        wt = w.float().view(N, taps, Cc).permute(0, 2, 1)
        y = torch.nn.functional.conv1d(xc, wt, bias, padding=halo, dilation=dil).transpose(1, 2)
        y = torch.nn.functional.leaky_relu(y, 0.1) * 0.5 + res.data().float()
        km = (torch.arange(T, device=dev)[None] < lens[:, None])[:, :, None]
        y = y * km
        torch.cuda.synchronize()
        print(f"conv taps={taps} dil={dil}: tc-vs-simt {rel(oa.data(), ob.data()):.2e} tc-vs-torch {rel(oa.data(), y):.2e} out2 {rel(o2a.data(), o2b.data()):.2e}"
              f" halo-zero {float(oa.buf.float().abs().sum() - oa.data().float().abs().sum()):.1e}")
    x = Seq(2, 40, 128)
    x.buf.copy_((torch.randn(80, 128, device=dev) * 0.5).half())
    w = (torch.randn(256, 128, device=dev) * 0.1).half()
    g1 = ops.gemm(x, w, 256, None, glu=True)
    g2 = ops.gemm(x, w, 256, None, glu=True, ref=True)
    full = x.buf.float() @ w.float().t()
    gt = full[:, 0::2] * torch.sigmoid(full[:, 1::2])
    print(f"glu: tc-vs-simt {rel(g1.buf, g2.buf):.2e} tc-vs-torch {rel(g1.buf, gt):.2e}")


def stage_fbank():
    w = S.make_waveforms(3, 16000 * 2)
    ns = torch.tensor([32000, 20000, 32000], dtype=torch.int32)
    fb, frames = ops.fbank(w.to(dev), ns.to(dev), 198)
    torch.cuda.synchronize()
    for i in range(3):
        ref = o_fbank(w[i, :ns[i]])
        n = ref.shape[0]
        assert int(frames[i]) == n, (int(frames[i]), n)
        err = (fb[i, :n].float().cpu() - ref).abs().max().item()
        pad = fb[i, n:].float().abs().max().item() if n < 198 else 0.0
        print(f"fbank utt{i}: frames {n} max abs err {err:.3e} (values are standardised ~N(0,1)); pad max {pad}")


def stage_ln():
    B, T, D = 3, 37, 1024
    x = Seq(B, T, D)
    x.buf.copy_(torch.randn(B * T, D, device=dev).half())
    w, b = torch.randn(D, device=dev), torch.randn(D, device=dev)
    y = ops.layernorm(x, w, b)
    ref = torch.nn.functional.layer_norm(x.buf.float(), (D,), w, b, 1e-5)
    print(f"layernorm: {rel(y.buf, ref):.2e}")


def stage_attn():
    torch.manual_seed(1)
    B, H, S, M = 2, 4, 150, 256
    qkv = Seq(B, S, 3 * M, lens=torch.tensor([150, 97], dtype=torch.int32, device=dev))
    qkv.buf.copy_((torch.randn(B * S, 3 * M, device=dev)).half())
    relk = (torch.randn(73, 64, device=dev) * 0.125).half()
    for causal, rel_t in [(False, None), (True, None), (False, relk)]:
        out = ops.self_attention(qkv, H, causal=causal, rel_k=rel_t, rel_left=64, rel_right=8)
        q, k, v = [t.float().view(B, S, H, 64).transpose(1, 2) for t in qkv.buf.view(B, S, 3 * M).split(M, dim=2)]
        w = q @ k.transpose(2, 3)
        if rel_t is not None:
            idx = (torch.arange(S, device=dev)[None] - torch.arange(S, device=dev)[:, None]).clamp(-64, 8) + 64
            w = w + torch.einsum("nhsk,stk->nhst", q, rel_t.float()[idx])
        w = w * 0.125
        km = torch.arange(S, device=dev)[None] < qkv.lens[:, None]
        w = w.masked_fill(~km[:, None, None, :], float("-inf"))
        if causal:
            w = w.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=dev).tril(), float("-inf"))
        ref = (torch.softmax(w, -1) @ v).transpose(1, 2).reshape(B * S, M)
        print(f"attention causal={causal} shaw={rel_t is not None}: {rel(out.buf, ref):.2e}")


def stage_dwconv():
    B, T, Cc, k = 2, 45, 256, 31
    x = Seq(B, T, Cc)
    x.buf.copy_(torch.randn(B * T, Cc, device=dev).half())
    w = (torch.randn(Cc, k, device=dev) * 0.2).half()
    lw, lb = torch.randn(Cc, device=dev), torch.randn(Cc, device=dev)
    y = ops.dwconv_ln_silu(x, w, lw, lb, k)
    xc = torch.nn.functional.pad(x.buf.float().view(B, T, Cc).transpose(1, 2), (k - 1, 0))
    c = torch.nn.functional.conv1d(xc, w.float().view(Cc, 1, k), groups=Cc).transpose(1, 2)
    ref = torch.nn.functional.silu(torch.nn.functional.layer_norm(c, (Cc,), lw, lb, 1e-5))
    print(f"dwconv_ln_silu: {rel(y.buf, ref.reshape(B * T, Cc)):.2e}")


def _tiny(dur=True):
    cfg, vc = C.tiny_v2(), C.tiny_vocoder()
    kw = dict(dur_gain=1.0, dur_bias=0.9) if dur else {}
    sd = S.make_unity_state_dict(cfg, 0, dec_gain=4.0, **kw)
    vsd = S.make_vocoder_state_dict(vc, 1)
    toks = S.make_tokenizers(cfg)
    return cfg, vc, sd, vsd, toks


def stage_e2e():
    from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model

    cfg, vc, sd, vsd, toks = _tiny()
    waves = S.make_waveforms(3, 32000)
    uo, vo = UnityOracle(cfg.to_dict(), sd, toks), VocoderOracle(vc.to_dict(), vsd)
    trace = {}
    ref = s2st(uo, vo, waves, "spa", 25, 45, hard_max=24, trace=trace)
    model = load_unity_model("tiny_v2", state_dict=sd, tokenizers=toks)
    voc = load_vocoder_model("tiny", state_dict=vsd)
    tr = Translator(model, voc, device="cuda")
    src = tr.fbank_batch(waves)
    print("fbank err", (src["seqs"].float().cpu() - ref["fbank"]).abs().max().item())
    eng = model.engine
    enc, lens, inner = eng.encode_speech(src["seqs"], None, return_inner=True)
    o_enc, _, o_inner = uo.encode_speech(ref["fbank"], None, return_inner=True)
    print("conformer inner rel err", rel(inner.buf.view(3, -1, cfg.model_dim), o_inner))
    print("encoder out rel err", rel(enc.buf.view(3, -1, cfg.model_dim), o_enc))
    opts = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=24)
    t0 = time.time()
    texts, speech = tr.predict(src, "s2st", "spa", text_generation_opts=opts)
    torch.cuda.synchronize()
    print("predict time", time.time() - t0)
    gen = Translator._last_generator
    hyps = gen.last_text_output.hypotheses
    for i in range(3):
        print(f"sent {i}: ids equal {hyps[i][0][1] == ref['text_ids'][i]}; score {hyps[i][0][0]:.4f} vs {ref['hyps'][i][0][0]:.4f}")
        if hyps[i][0][1] != ref["text_ids"][i]:
            print("   gpu", hyps[i][0][1])
            print("   ref", ref["text_ids"][i])
    print("texts equal", texts == ref["texts"], texts[0][:50])
    uout = gen.last_unit_output
    d = uout["dec_out"]
    print("teacher-forced dec_out rel err", rel(d.buf.view(d.B, d.T, -1), ref["dec_out"]))
    print("char_lens equal", torch.equal(uout["char_lens"].cpu().long(), ref["chars"][2]))
    print("dur equal", torch.equal(uout["dur"].cpu().long(), ref["dur"]), "unit_lens", uout["unit_lens"].tolist(), ref["unit_lens"].tolist())
    for i in range(3):
        print(f"units[{i}] equal", speech.units[i] == ref["speech_units"][i], len(speech.units[i]))
        if speech.units[i] != ref["speech_units"][i]:
            a, b = speech.units[i], ref["speech_units"][i]
            nd = sum(x != y for x, y in zip(a, b))
            print("   differing positions:", nd, "of", len(b))
    for i in range(3):
        w, r = speech.audio_wavs[i].float().cpu(), ref["wavs"][i]
        if w.shape == r.shape:
            print(f"wav[{i}] max abs err {(w - r).abs().max().item():.3e} (signal std {r.std().item():.3f})")
        else:
            print("wav shape mismatch", w.shape, r.shape)


def stage_vocoder():
    from seamless_communication_b200.models.vocoder import load_vocoder_model

    _, vc, _, vsd, _ = _tiny()
    voc = load_vocoder_model("tiny", state_dict=vsd)
    g = torch.Generator().manual_seed(3)
    units = torch.randint(0, vc.num_embeddings, (2, 23), generator=g)
    wav = voc(units.to(dev), "spa", -1, dur_prediction=False)
    ref = VocoderOracle(vc.to_dict(), vsd)(units, [25, 25], [45, 45])
    torch.cuda.synchronize()
    print("vocoder wav", tuple(wav.shape), f"max abs err {(wav.float().cpu() - ref).abs().max().item():.3e} (std {ref.std().item():.3f})")


def stage_iso():
    """Feed the oracle's intermediates into each GPU stage (isolates numerical drift from logic errors)."""
    from seamless_communication_b200.models.unity import load_unity_model

    cfg, vc, sd, vsd, toks = _tiny()
    waves = S.make_waveforms(3, 32000)
    uo = UnityOracle(cfg.to_dict(), sd, toks)
    trace = {"sentence": 1}
    ref = s2st(uo, VocoderOracle(vc.to_dict(), vsd), waves, "spa", 25, 45, hard_max=24, trace=trace)
    model = load_unity_model("tiny_v2", state_dict=sd, tokenizers=toks)
    eng = model.engine
    M = cfg.model_dim
    enc = Seq(3, ref["enc"].shape[1], M, buf=ref["enc"].to(dev).half().reshape(-1, M).contiguous())
    ts = ref["text_seqs"].to(dev)
    tl = torch.tensor([len(s) - 1 for s in ref["text_ids"]], dtype=torch.int32, device=dev)
    dec = eng.decode_full(ts, tl, enc, None)
    print("decode_full(oracle ids, oracle enc) rel err", rel(dec.buf.view(3, -1, M), ref["dec_out"]))
    # teacher-forced logits of the oracle's best hypothesis vs oracle logits
    lg = ops.gemm_raw(dec.buf, eng.w["text_embed"], cfg.text_vocab, out_f32=True).view(3, -1, cfg.text_vocab)
    olg = uo.project(ref["dec_out"])
    print("teacher-forced logits max abs err", (lg.float().cpu() - olg).abs().max().item(), "logit std", olg.std().item())
    # beam search from the oracle's encoder output
    hyps = eng.beam_search(enc, None, [cfg.text_eos, toks[0].lang_index("spa")], beam=5, hard_max=24)
    for i in range(3):
        same = hyps[i][0][1] == ref["text_ids"][i]
        print(f"beam(oracle enc) sent {i}: equal {same} score {hyps[i][0][0]:.4f} vs {ref['hyps'][i][0][0]:.4f}; n_fin {len(hyps[i])} vs {len(ref['hyps'][i])}")
        if not same:
            # margin audit: score the GPU hypothesis with the oracle
            ids = torch.tensor(hyps[i][0][1])[None]
            h = uo.decoder(uo.embed_text(ids[:, :-1], 0), ref["enc"][i:i + 1], None)
            lp = torch.log_softmax(uo.project(h).float(), -1)[0]
            sc = sum(float(lp[t, ids[0, t + 1]]) for t in range(ids.shape[1] - 1)) / (ids.shape[1] - 1)
            print(f"   oracle score of GPU hyp {sc:.4f} vs oracle best {ref['hyps'][i][0][0]:.4f}")
            print("   gpu", hyps[i][0][1]); print("   ref", ref["text_ids"][i])
    # T2U from the oracle's decoder output, free-running durations and oracle durations
    dseq = Seq(3, ref["dec_out"].shape[1], M, lens=tl, buf=ref["dec_out"].to(dev).half().reshape(-1, M).contiguous())
    units, ulens, aux = eng.t2u(dseq, ts)
    print("t2u_enc rel err", rel(aux["t2u_enc"].buf.view(3, -1, M), ref["t2u_enc"]))
    print("char_lens equal", torch.equal(aux["char_lens"].cpu().long(), ref["chars"][2]), "char_seq_lens", aux["char_seq_lens"].tolist(), ref["chars"][1].tolist())
    cs = ref["chars"][0]
    print("char_seqs equal", torch.equal(aux["char_seqs"].cpu().long()[:, :cs.shape[1]], cs))
    nd = (aux["dur"].cpu().long() != ref["dur"]).sum().item()
    print("durations differing", nd, "of", ref["dur"].numel(), "unit_lens", ulens.tolist(), ref["unit_lens"].tolist())
    units2, ulens2, aux2 = eng.t2u(dseq, ts, durations=ref["dur"])
    z = aux2["fft_out"]
    print("fft_out (oracle durations) rel err", rel(z.data(), ref["fft_out"]))
    for i in range(3):
        n = int(ref["unit_lens"][i])
        a, b = units2[i, :n].cpu(), ref["units"][i, :n]
        print(f"units (oracle durations) sent {i}: differing {(a != b).sum().item()} of {n}")


STAGES = dict(iso=stage_iso, gemm=stage_gemm, fbank=stage_fbank, ln=stage_ln, attn=stage_attn, dwconv=stage_dwconv, vocoder=stage_vocoder,
              e2e=stage_e2e)

if __name__ == "__main__":
    names = sys.argv[1:] or list(STAGES)
    print(torch.cuda.get_device_name(0))
    for n in names:
        print(f"==== {n}")
        try:
            STAGES[n]()
            torch.cuda.synchronize()
        except Exception:
            traceback.print_exc()
            try:
                torch.cuda.synchronize()
            except Exception as e:  # sticky CUDA error: stop
                print("CUDA context broken:", e)
                break
