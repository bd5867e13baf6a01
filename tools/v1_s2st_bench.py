#!/usr/bin/env python
"""Per-stage times of speech-to-speech on seamlessM4T_large (arch `base`, autoregressive T2U) + vocoder_36langs, with
seeded random-init weights, on a batch of 10 s utterances (default 32 x 160000 samples):
  encoder -> text search (beam 5, hard_max 102) -> T2U encoder -> unit search (beam 5) -> vocoder (duration prediction).
Random weights rarely emit EOS, so the unit search length is set explicitly (--unit-positions, default 250 and 500) and
every hypothesis runs to it; the text search runs to its hard_max for the same reason.

For the unit search the script prints ms per step next to the bytes one step has to read, computed from the shapes:
  * weights: per layer q|k|v, self out, cross q, cross out (6 M^2) and the FFN (2 M F), fp16, plus the tied projection
    (V x M) - 6 x 46 MB + 20.6 MB at base;
  * cross K/V: layers x B x S_enc x 2M fp16 (S_enc = the bucketed text length: the step reads every row of it);
  * self K/V at position t: layers x B x beam x t x 2M fp16 (3.93 MB per position at 32 x beam 5), averaged over the
    search as t = positions / 2.
These are computed bytes, not measured traffic.  Times are CUDA-event medians over --iters runs after one warm-up run.
The vocoder takes the whole batch (Vocoder.forward with duration prediction, as Translator.predict calls it); random
weights give about 4 frames per unit, so at 500 units it generates the batch in parts (VocoderEngine.resynthesize
splits a batch whose frames exceed one sb_gemm grid).
Also prints the card's name and power limit."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import config as C, ops, synthetic as S  # noqa: E402
from seamless_communication_b200.models.unity import UnitTokenizer, load_unity_model  # noqa: E402
from seamless_communication_b200.models.vocoder import load_vocoder_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--arch", default="seamlessM4T_large")
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--samples", type=int, default=160000)
ap.add_argument("--text-hard-max", type=int, default=102)
ap.add_argument("--unit-positions", type=int, nargs="+", default=[250, 500])
ap.add_argument("--iters", type=int, default=3)
args = ap.parse_args()
dev = "cuda"
LANG = "spa"
BEAM = 5


def timed(fn, iters):
    """fn() once to warm up (graph capture, state allocation), then the median / min / max of `iters` timed calls."""
    fn()
    ms = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), min(ms), max(ms)


def line(name, t, extra=""):
    med, lo, hi = t
    print(f"{name:30s} median {med:9.2f} ms (min {lo:9.2f}, max {hi:9.2f}) {extra}", flush=True)


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
with torch.inference_mode():
    cfg = C.UNITY_ARCHS[C.MODEL_CARDS.get(args.arch, args.arch)]()
    model = load_unity_model(args.arch, synthetic=True, seed=0)
    eng, t2u = model.engine, model.t2u_model
    voc = load_vocoder_model("vocoder_36langs", synthetic=True)
    B = args.batch
    waves = S.make_waveforms(B, args.samples, seed=5).to(dev)
    T_fb = 1 + (args.samples - 400) // 160
    fb, frames = ops.fbank(waves, torch.full((B,), args.samples, dtype=torch.int32, device=dev), T_fb + T_fb % 2)
    fb16 = fb.to(torch.float16)
    print(f"{args.arch} (arch {cfg.name}) + vocoder_36langs, batch {B} x {args.samples} samples, beam {BEAM}")

    st = {}

    def encoder():
        st["enc"], st["enc_lens"] = eng.encode_speech(fb16, frames)

    def text_search():
        tok = eng.text_tokenizer
        prefix = tok.create_encoder(task="translation", lang=LANG, mode="target").prefix_indices.tolist()
        st["hyps"] = eng.beam_search(st["enc"], st["enc_lens"], prefix, beam=BEAM, soft_max=(1, 200),
                                     hard_max=args.text_hard_max)
        lens = [len(h[0][1]) - 1 for h in st["hyps"]]
        st["dec"] = eng.harvest_decoder_states(lens)
        st["text_lens"] = torch.tensor(lens, dtype=torch.int32, device=dev)

    def t2u_encoder():
        st["t2u_enc"] = eng.t2u_encode(st["dec"])

    line("encoder", timed(encoder, args.iters))
    line("text search (+ state harvest)", timed(text_search, args.iters),
         f"text length {max(len(h[0][1]) for h in st['hyps'])}")
    line("T2U encoder", timed(t2u_encoder, args.iters))

    M, F, V, Lr = cfg.model_dim, cfg.t2u_ffn_dim, cfg.unit_vocab, cfg.t2u_dec_layers
    S_enc = st["t2u_enc"].T
    S_b = -(-S_enc // t2u.S_ENC_BUCKET) * t2u.S_ENC_BUCKET
    w_bytes = Lr * (6 * M * M + 2 * M * F) * 2 + V * M * 2
    cross_bytes = Lr * B * S_b * 2 * M * 2
    per_pos = Lr * B * BEAM * 2 * M * 2
    print(f"unit step weights {w_bytes / 1e6:.1f} MB, cross K/V {cross_bytes / 1e6:.1f} MB (S_enc {S_enc} -> {S_b}), "
          f"self K/V {per_pos / 1e6:.2f} MB per position")
    prefix = UnitTokenizer(cfg.num_units, cfg.unit_langs, cfg.name).create_encoder(LANG).prefix_indices.tolist()
    for n in args.unit_positions:
        def unit_search():
            st["unit_hyps"] = t2u.beam_search(st["t2u_enc"], st["text_lens"], prefix, beam=BEAM, soft_max=(0, 0), hard_max=n)

        t = timed(unit_search, args.iters)
        steps = n - 1  # one bootstrap step for the language token, then n - 2 search steps
        got = max(len(h[0][1]) for h in st["unit_hyps"])
        step_bytes = w_bytes + cross_bytes + per_pos * n / 2
        line(f"unit search {n} positions", t,
             f"{t[0] / steps:.3f} ms/step; computed {step_bytes / 1e6:.0f} MB/step (self K/V {per_pos * n / 2 / 1e6:.0f} MB "
             f"at the mean position) -> {step_bytes / (t[0] / steps) / 1e6:.0f} GB/s; hypothesis length {got}")

        # the vocoder input of each row as the generator and the translator build it: the hypothesis without its
        # [eos, lang] prefix, units shifted by the 4 control symbols, the final EOS turned into 1
        units = torch.tensor([[u - 4 for u in h[0][1][2:-1]] + [1] for h in st["unit_hyps"]], device=dev)

        def vocoder():
            voc(units, LANG, -1, dur_prediction=True)

        line(f"vocoder ({units.shape[1]} units / row)", timed(vocoder, args.iters),
             f"{int(voc.last_wav_lens.max()) / 16000:.2f} s of audio in the longest row")
