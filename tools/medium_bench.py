#!/usr/bin/env python
"""seamlessM4T_medium against seamlessM4T_large, fp16 and FP8 decoder weights, in one process on seeded synthetic
weights, on the BASELINE workload: 32 utterances x 10 s, beam 5, text hard_max 102.

For each of the four models, alternated round by round (--rounds), it times with CUDA events:
  * S2ST `Translator.predict` (unit search: beam 5, hard_max --unit-hard-max; random weights rarely emit EOS, so the
    unit search runs to that budget) with vocoder_36langs, in utterances per second;
  * S2TT `Translator.predict`, in utterances per second;
  * the text beam search alone on the batch's encoder output, in ms per step,
next to the bytes one text-search step has to read, computed from the shapes (not measured traffic):
  * decoder weights: per layer q|k|v, self out, cross q, cross out (6 M^2) and the FFN (2 M F), 2 bytes each in fp16,
    1 in FP8;
  * the tied projection: V x M, 2 bytes in fp16, 1 in FP8;
  * self K/V at the mean position t = hard_max / 2: layers x 160 rows x t x 2M fp16;
  * cross K/V: layers x 32 x S_enc x 2M fp16.
Every model runs once before the first timed round (graph capture, state allocation).  Prints the card's name and power
limit, and one JSON line with the medians."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import config as C, synthetic as S  # noqa: E402
from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator  # noqa: E402
from seamless_communication_b200.models.unity import load_unity_model  # noqa: E402
from seamless_communication_b200.models.vocoder import load_vocoder_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--cards", nargs="+", default=["seamlessM4T_medium", "seamlessM4T_large"])
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--samples", type=int, default=160000)
ap.add_argument("--text-hard-max", type=int, default=102)
ap.add_argument("--unit-hard-max", type=int, default=250)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--no-fp8", action="store_true")
args = ap.parse_args()
dev = "cuda"
LANG, BEAM = "spa", 5


def event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def step_bytes(cfg, fp8, S_enc):
    M, F, L, V = cfg.model_dim, cfg.dec_ffn_dim, cfg.dec_layers, cfg.text_vocab
    wb = 1 if fp8 else 2
    R, t = args.batch * BEAM, args.text_hard_max / 2
    return {"weights": L * (6 * M * M + 2 * M * F) * wb, "projection": V * M * wb,
            "self_kv": L * R * t * 2 * M * 2, "cross_kv": L * args.batch * S_enc * 2 * M * 2}


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}", flush=True)
text_opts = SequenceGeneratorOptions(beam_size=BEAM, soft_max_seq_len=(1, 200), hard_max_seq_len=args.text_hard_max)
unit_opts = SequenceGeneratorOptions(beam_size=BEAM, soft_max_seq_len=(25, 50), hard_max_seq_len=args.unit_hard_max)
with torch.inference_mode():
    voc = load_vocoder_model("vocoder_36langs", synthetic=True)
    models = {}
    for name in args.cards:
        cfg = C.UNITY_ARCHS[C.MODEL_CARDS[name]]()
        sd = S.make_unity_state_dict(cfg, 0, with_t2u=True)
        toks = S.make_tokenizers(cfg)
        for dt in ([torch.float16] if args.no_fp8 else [torch.float16, torch.float8_e4m3fn]):
            tag = f"{name} {'fp8' if dt != torch.float16 else 'fp16'}"
            models[tag] = (cfg, dt != torch.float16,
                           Translator(load_unity_model(name, state_dict=sd, tokenizers=toks, decoder_weight_dtype=dt), voc, device=dev))
        del sd
    waves = S.make_waveforms(args.batch, args.samples, seed=5)
    B = args.batch
    print(f"batch {B} x {args.samples} samples, beam {BEAM}, text hard_max {args.text_hard_max}, "
          f"unit hard_max {args.unit_hard_max}", flush=True)

    def runs(tr):
        src = tr.fbank_batch(waves)
        eng = tr.model.engine
        enc, enc_lens = eng.encode_speech(src["seqs"].to(torch.float16), src["seq_lens"])
        prefix = tr.text_tokenizer.create_encoder(task="translation", lang=LANG, mode="target").prefix_indices.tolist()
        return {"s2st": lambda: tr.predict(src, "s2st", LANG, text_generation_opts=text_opts, unit_generation_opts=unit_opts),
                "s2tt": lambda: tr.predict(src, "s2tt", LANG, text_generation_opts=text_opts),
                "text_search": lambda: eng.beam_search(enc, enc_lens, prefix, beam=BEAM, soft_max=(1, 200),
                                                       hard_max=args.text_hard_max)}, enc.T

    fns, s_enc = {}, {}
    for tag, (cfg, fp8, tr) in models.items():
        fns[tag], S_enc = s_enc[tag] = runs(tr)
        for f in fns[tag].values():
            f()  # warm-up
        b = step_bytes(cfg, fp8, S_enc)
        print(f"{tag}: {cfg.dec_layers} decoder layers, FFN {cfg.dec_ffn_dim}, V {cfg.text_vocab}; computed bytes per text step: "
              + ", ".join(f"{k} {v / 1e9:.3f} GB" for k, v in b.items()) + f" (S_enc {S_enc})", flush=True)
    times = {tag: {k: [] for k in f} for tag, f in fns.items()}
    steps = {}
    for r in range(args.rounds):
        for tag, f in fns.items():
            for k, fn in f.items():
                ms, out = event_ms(fn)
                times[tag][k].append(ms)
                if k == "text_search":
                    steps[tag] = max(len(h[0][1]) for h in out) - 2  # positions after the 2-token prefix
    result = {"card": card}
    for tag, t in times.items():
        cfg, fp8, _ = models[tag]
        med = {k: statistics.median(v) for k, v in t.items()}
        n = steps[tag]
        gb = sum(step_bytes(cfg, fp8, s_enc[tag][1]).values()) / 1e9
        result[tag] = {"s2st_utt_per_s": B / med["s2st"] * 1e3, "s2tt_utt_per_s": B / med["s2tt"] * 1e3,
                       "text_ms_per_step": med["text_search"] / n, "text_steps": n,
                       "text_step_computed_gb": gb,
                       "spread_ms": {k: [round(min(v), 1), round(max(v), 1)] for k, v in t.items()}}
        print(f"{tag:30s} S2ST {result[tag]['s2st_utt_per_s']:7.1f} utt/s  S2TT {result[tag]['s2tt_utt_per_s']:7.1f} utt/s  "
              f"text search {med['text_search']:8.1f} ms = {result[tag]['text_ms_per_step']:.3f} ms/step over {n} steps "
              f"({gb:.2f} GB computed per step)  "
              f"(min/max ms {result[tag]['spread_ms']})", flush=True)
    print(json.dumps(result))
