#!/usr/bin/env python
"""Cost of n-gram repeat blocking (NGramRepeatBlockProcessor) at the bench shape: seamlessM4T_v2_large + vocoder_v2 with
seeded random-init weights, a batch of 32 x 10 s synthetic utterances, beam 5, hard_max_seq_len 102 (160 rows).

1. The select half of one search step (CUDA-graph replay): without blocking (g_sel: top-K, sb_beam_step,
   sb_step_advance) and with blocking at n = 2, 3, 4 (g_sel_ngram: sb_ngram_ban_step first, then the `_ban` top-K).
   CUDA events around each replay; before every replay, outside the timed window, the rows are restored to those of
   a finished search and the step index is set to the same position.  Two row contents: the search's own rows, and the
   worst case of every row one repeated token (every start matches: t - n + 2 bans per row).
2. Translator.predict end to end (host clock around a device synchronise), S2TT and S2ST, with blocking off and on at
   the reference CLI's default `--no_repeat_ngram_size 4`.

Medians over --iters runs after one warm-up run.  Prints the card's name and power limit."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import config as C, synthetic as S  # noqa: E402
from seamless_communication_b200.inference import NGramRepeatBlockProcessor, SequenceGeneratorOptions, Translator  # noqa: E402
from seamless_communication_b200.models.unity import load_unity_model  # noqa: E402
from seamless_communication_b200.models.vocoder import load_vocoder_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--replays", type=int, default=200)
ap.add_argument("--ngram", type=int, default=4, help="n of the end-to-end runs")
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card)
cfg, vc = C.base_v2(), C.base_vocoder()
toks = S.make_tokenizers(cfg)
model = load_unity_model("seamlessM4T_v2_large", device="cuda", state_dict=S.make_unity_state_dict(cfg, seed=0, dec_gain=4.0),
                         tokenizers=toks)
voc = load_vocoder_model("vocoder_v2", device="cuda", state_dict=S.make_vocoder_state_dict(vc, seed=1))
plain = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=102)
blocked = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=102,
                                   step_processor=NGramRepeatBlockProcessor(args.ngram))
tr = Translator(model, voc, device="cuda")
src = tr.fbank_batch(S.make_waveforms(args.batch, 160000, seed=1234).cuda())
tr.predict(src, "s2tt", "spa", text_generation_opts=plain)
eng = model.engine
st = eng._last_search_state
STEP = 60

# ---- 1. select half per step
search_rows = st["seqs"].clone()
equal_rows = search_rows.clone()
equal_rows[:, 2:] = 7


def time_select(graph, rows):
    ts = []
    for _ in range(args.replays):
        st["seqs"].copy_(rows)
        st["step"].fill_(STEP)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        ts.append((e0, e1))
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) * 1e3 for a, b in ts)


with torch.inference_mode():
    graphs = [("no blocking (g_sel)", st["g_sel"])]
    for n in (2, 3, 4):
        eng._set_ngram(st, n)
        eng._capture_ngram(st)
        graphs.append((f"n = {n} (g_sel_ngram)", st["g_sel_ngram"]))
    print(f"select per step at step {STEP}, {st['R']} rows (us, median of {args.replays}):   search rows   all one token")
    for name, g in graphs:
        time_select(g, search_rows)  # warm-up
        print(f"  {name:24s} {time_select(g, search_rows):12.1f} {time_select(g, equal_rows):14.1f}")

# ---- 2. predict end to end
print(f"Translator.predict, {args.batch} x 10 s (ms, median of {args.iters}), blocking at n = {args.ngram}:")
for task in ("s2tt", "s2st"):
    out = {}
    for name, opts in (("off", plain), ("on", blocked)):
        tr.predict(src, task, "spa", text_generation_opts=opts)
        ts = []
        for _ in range(args.iters):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            texts, _ = tr.predict(src, task, "spa", text_generation_opts=opts)
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        hyps = [h[0][1] for h in Translator._tls.generator.last_text_output.hypotheses]
        out[name] = (statistics.median(ts), texts, hyps)
    changed = sum(a != b for a, b in zip(out["on"][1], out["off"][1]))
    lens = [statistics.mean(len(h) for h in out[k][2]) for k in ("off", "on")]
    print(f"  {task}: off {out['off'][0]:8.1f}   on {out['on'][0]:8.1f}   rows whose text changed: {changed}/{args.batch}   "
          f"mean hypothesis length off {lens[0]:.1f}, on {lens[1]:.1f}")
