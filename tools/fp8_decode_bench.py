#!/usr/bin/env python
"""FP8 decoder weights against fp16, alternated in one session (DESIGN.md section 16).

  * each weight product of a decoder layer and the tied projection at 160 rows, in CUDA graphs that chain launches over
    24 different weight tensors (as tools/decode_gemm_bench.py / proj_bench.py), fp16 entry against e4m3 entry;
  * the forward half of one search step (the step's products, attention, LayerNorms and projection; its replayed graph)
    of seamlessM4T_v2_large at 32 sentences x beam 5;
  * Translator.predict S2ST over 32 x 10 s, beam 5, hard_max 102, with 1 lane and 4 lanes (LanePool): median of 3
    alternated runs;
  * the AR unit search of seamlessM4T_large (unit decoder only, 32 rows x beam 5, 250 positions).
It also checks that the FP8 bench batch equals an fp16 model of the dequantized weights bit for bit, and reports
divergence statistics of the FP8 model from the fp16 model of the original synthetic weights: the teacher-forced logit
difference on the fp16 model's hypotheses and the share of identical hypotheses.  These say how far the weight rounding
moves the outputs of random weights; they are not a quality measure.
Prints the card and its power limit with the numbers; --json writes them too."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import config as C, ops, synthetic as S  # noqa: E402
from seamless_communication_b200.models.fp8_weights import dequantize_decoder_weights, quantize_rows  # noqa: E402
from seamless_communication_b200.ops import ACT_RELU, Seq  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--json", default=None)
ap.add_argument("--skip-unit", action="store_true", help="leave out the seamlessM4T_large unit search")
args = ap.parse_args()
dev = "cuda"
out = {}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def graph_us(fn, n_calls, reps=20):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(3):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * n_calls)


# ---------------------------------------------------------------------------------------------- products, projection
R, LAYERS, M, FFN, V = 160, 24, 1024, 8192, 256102
S_QKV, S_ATT, S_FFN = ops.decode_splits(R, M, FFN)
out["card"] = card()
print("card, power limit:", out["card"])
prod = {}
for name, n, k, splits in (("qkv", 3 * M, M, S_QKV), ("attn_out", M, M, S_ATT), ("ffn_inner", FFN, M, 0), ("ffn_out", M, FFN, S_FFN)):
    a = Seq(1, R, k)
    a.buf.normal_()
    ws = [(torch.randn(n, k, device=dev) * 0.02) for _ in range(LAYERS)]
    qs = [quantize_rows(w) for w in ws]
    ws = [w.half() for w in ws]
    bias = torch.zeros(n, device=dev)
    part = torch.empty(max(splits, 1) * ops.slice_rows(R), n, device=dev)
    o = Seq(1, R, n)

    def f16():
        for w in ws:
            if splits:
                ops.gemm_splitk(a, w, n, splits, part, transposed=True)
            else:
                ops.gemm_decode(a, w, n, bias, act=ACT_RELU, out=o)

    def f8():
        for q, s in qs:
            if splits:
                ops.gemm_splitk_e4m3(a, q, s, n, splits, part)
            else:
                ops.gemm_decode_e4m3(a, q, s, n, bias, act=ACT_RELU, out=o)
    t = {"fp16": [], "fp8": []}
    for _ in range(3):
        t["fp16"].append(graph_us(f16, LAYERS))
        t["fp8"].append(graph_us(f8, LAYERS))
    prod[name] = {kk: min(v) for kk, v in t.items()}
    prod[name]["weight_MB_fp16"] = n * k * 2 / 1e6
    del ws, qs
h = Seq(1, R, M)
h.buf.normal_()
E = torch.randn(V, M, device=dev) * 0.02
qE, sE = quantize_rows(E)
E = E.half()
logits = Seq(1, R, V, dtype=torch.float32, buf=torch.empty((R, (V + 7) // 8 * 8), device=dev))
stats = torch.empty(((V + 127) // 128, R, 2), device=dev)
t = {"fp16": [], "fp8": []}
for _ in range(3):
    t["fp16"].append(graph_us(lambda: [ops.gemm(h, E, V, None, out=logits, out_f32=True, tile_stats=stats) for _ in range(4)], 4))
    t["fp8"].append(graph_us(lambda: [ops.vocab_proj_e4m3(h, qE, sE, V, logits, stats) for _ in range(4)], 4))
prod["projection"] = {kk: min(v) for kk, v in t.items()}
prod["projection"]["weight_MB_fp16"] = V * M * 2 / 1e6
del E, qE, sE, logits, stats
out["kernels_us"] = prod
for k, v in prod.items():
    print(f"{k:11s} fp16 {v['fp16']:8.1f} us  fp8 {v['fp8']:8.1f} us  ({v['weight_MB_fp16']:.1f} MB fp16 weights)")

# ---------------------------------------------------------------------------------------------- whole models
from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator  # noqa: E402
from seamless_communication_b200.models.unity import load_unity_model  # noqa: E402
from seamless_communication_b200.models.vocoder import load_vocoder_model  # noqa: E402
from seamless_communication_b200.parallel import LanePool  # noqa: E402

cfg, vc = C.base_v2(), C.base_vocoder()
sd = S.make_unity_state_dict(cfg, seed=0, dec_gain=4.0)
toks = S.make_tokenizers(cfg)
voc = load_vocoder_model("vocoder_v2", device=dev, state_dict=S.make_vocoder_state_dict(vc, seed=1))
trs = {"fp16": Translator(load_unity_model("seamlessM4T_v2_large", device=dev, state_dict=sd, tokenizers=toks), voc, device=dev),
       "fp8": Translator(load_unity_model("seamlessM4T_v2_large", device=dev, state_dict=sd, tokenizers=toks,
                                          decoder_weight_dtype=torch.float8_e4m3fn), voc, device=dev),
       "fp16_dequantized": Translator(load_unity_model("seamlessM4T_v2_large", device=dev, tokenizers=toks,
                                                       state_dict=dequantize_decoder_weights(sd, cfg)), voc, device=dev)}
del sd
waves = S.make_waveforms(32, 160000, seed=1234).to(dev)
opts = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=102)


def predict(tr):
    return tr.predict(tr.fbank_batch(waves), "s2st", "spa", text_generation_opts=opts)


res = {k: predict(tr) for k, tr in trs.items()}
same = res["fp8"][0] == res["fp16_dequantized"][0] and res["fp8"][1].units == res["fp16_dequantized"][1].units and all(
    torch.equal(a, b) for a, b in zip(res["fp8"][1].audio_wavs, res["fp16_dequantized"][1].audio_wavs))
out["fp8_equals_fp16_on_dequantized_bench_batch"] = bool(same)
print("FP8 bench batch equals the fp16 model of the dequantized weights bit for bit:", same)

# divergence statistics against the original weights (not a quality measure)
ident = sum(a == b for a, b in zip(res["fp16"][0], res["fp8"][0])) / len(res["fp16"][0])
eng16, eng8 = trs["fp16"].model.engine, trs["fp8"].model.engine
div = {"identical_texts_share": ident}
# teacher-forced: the fp16 model's best hypotheses through both decoders, on the fp16 model's encoder output
st = eng16._last_search_state
if st is not None:
    fin = st["fin"]
    best = st["best_fin"]
    B = st["B"]
    seqs = [fin["seqs"][b, max(best[b], 0), :int(fin["len"][b, max(best[b], 0)])].tolist() for b in range(B)]
    L = max(len(s) for s in seqs) - 1
    tin = torch.tensor([s[:-1] + [0] * (L - len(s) + 1) for s in seqs], device=dev)
    tl = torch.tensor([len(s) - 1 for s in seqs], dtype=torch.int32, device=dev)
    from seamless_communication_b200.ops import gemm_raw  # noqa: E402
    with torch.inference_mode():
        # the bench batch's encoder output, as the cross-attention K/V of the fp16 search (not quantized: the same in both)
        e = Seq(B, st["S_enc"], M, buf=torch.empty((1, M), dtype=torch.float16, device=dev))
        d16 = eng16.decode_full(tin, tl, e, st["enc_lens"], cross_kv=st["cross_kv"])
        d8 = eng8.decode_full(tin, tl, e, st["enc_lens"], cross_kv=st["cross_kv"])
        l16 = gemm_raw(d16.buf, eng16.w["text_embed"], cfg.text_vocab, out_f32=True)
        l8 = gemm_raw(d8.buf, eng8.w["text_embed"], cfg.text_vocab, out_f32=True)
        mask = (torch.arange(L, device=dev)[None, :] < tl[:, None]).reshape(-1)
        dl = (l16 - l8)[mask].abs()
        div.update(logit_abs_diff_max=dl.max().item(), logit_abs_diff_mean=dl.mean().item(),
                   logit_abs_mean=l16[mask].abs().mean().item(),
                   argmax_agreement=(l16[mask].argmax(-1) == l8[mask].argmax(-1)).float().mean().item())
out["divergence_not_quality"] = div
print("divergence from the fp16 model of the original weights (not a quality measure):", json.dumps(div))

# forward half of one search step: the replayed g_fwd graph of the bench state (the step index is not advanced)
step = {}
for k in ("fp16", "fp8"):
    st = trs[k].model.engine._last_search_state
    step[k] = []
for _ in range(3):
    for k in ("fp16", "fp8"):
        st = trs[k].model.engine._last_search_state
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st["g_fwd"].replay()
        e0.record()
        for _ in range(20):
            st["g_fwd"].replay()
        e1.record()
        torch.cuda.synchronize()
        step[k].append(e0.elapsed_time(e1) / 20)
out["step_forward_ms"] = {k: min(v) for k, v in step.items()}
print("search step, forward half (ms):", out["step_forward_ms"])

# predict, 1 and 4 lanes, median of 3 alternated runs
pred = {}
for lanes in (1, 4):
    pools = {k: (LanePool(dev, lanes, [trs[k].model.engine]) if lanes > 1 else None) for k in ("fp16", "fp8")}
    times = {"fp16": [], "fp8": []}

    def run(k, n):
        pool = pools[k]
        if pool is None:
            for _ in range(n):
                predict(trs[k])
            return
        futs = [pool.submit(i, predict, trs[k]) for i in range(n)]
        for f in futs:
            _, done = f.result()
            torch.cuda.current_stream().wait_event(done)
    for k in ("fp16", "fp8"):
        if pools[k] is not None:
            pools[k].warm(lambda k=k: predict(trs[k]))
        run(k, lanes)
    n = 4 * lanes
    for _ in range(3):
        for k in ("fp16", "fp8"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(k, n)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3 / n)
    for p in pools.values():
        if p is not None:
            p.close()
    pred[f"lanes{lanes}"] = {k: statistics.median(v) for k, v in times.items()}
    print(f"predict S2ST 32 x 10 s, {lanes} lane(s), ms per batch (median of 3):", pred[f"lanes{lanes}"])
out["predict_ms_per_batch"] = pred
del trs, res

# AR unit search of seamlessM4T_large: the unit decoder only, 250 positions
if not args.skip_unit:
    from seamless_communication_b200.engine import UnitYEngine  # noqa: E402
    from seamless_communication_b200.models.unity.model import t2u_decoder_config, t2u_decoder_state_dict  # noqa: E402
    big = C.base()
    usd = t2u_decoder_state_dict(S.make_unity_state_dict(big, seed=0, dec_gain=4.0, with_t2u=True))
    ucfg = t2u_decoder_config(big)
    engs = {"fp16": UnitYEngine(ucfg, usd, (None, None), device=dev),
            "fp8": UnitYEngine(ucfg, usd, (None, None), device=dev, decoder_weight_dtype=torch.float8_e4m3fn)}
    del usd
    x = torch.randn(32 * 64, M, device=dev).half()
    enc = Seq(32, 64, M, buf=x)
    times = {"fp16": [], "fp8": []}
    for k in engs:
        engs[k].beam_search(enc, None, [ucfg.text_eos, 5], beam=5, soft_max=(0, 0), hard_max=250)
    for _ in range(3):
        for k in engs:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            engs[k].beam_search(enc, None, [ucfg.text_eos, 5], beam=5, soft_max=(0, 0), hard_max=250)
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    steps = {k: int(e._last_search_state["step"].item()) for k, e in engs.items()}
    out["unit_search_ms"] = {k: statistics.median(v) for k, v in times.items()}
    out["unit_search_steps"] = steps
    print("AR unit search, 32 x beam 5, hard_max 250 (ms, median of 3):", out["unit_search_ms"], "steps run:", steps)

if args.json:
    with open(args.json, "w") as f:
        json.dump(out, f, indent=1)
