#!/usr/bin/env python
"""Time unit resynthesis with the vocoder's duration predictor (Vocoder(..., dur_prediction=True)) on the `base` vocoder:
a batch of deduplicated unit rows (default 32 x 250 units) with the synthetic duration predictor (durations average
about 2), so each row expands to about 500 frames = 10 s of 16 kHz audio, with different lengths per row.

Reported, as CUDA-event time per call (median over --iters calls, after --warmup calls):
  * predictor + expansion: unit embedding, VariancePredictor, durations, the one host sync, HardUpsampling;
  * generator: the HiFi-GAN on the ragged batch, every row masked to its own length;
  * plain generator: the same rows expanded with repeat_interleave on the host (each padded to the longest row by
    repeating its last unit) through dur_prediction=False, embedding included.
Also prints audio seconds per call and the card's name and power limit."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import config as C, synthetic as S  # noqa: E402
from seamless_communication_b200.models.vocoder import load_vocoder_model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--units", type=int, default=250)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
args = ap.parse_args()

dev = "cuda"
vc = C.base_vocoder()
voc = load_vocoder_model("vocoder_v2", device=dev, state_dict=S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True))
eng = voc.code_generator
B, U = args.batch, args.units
g = torch.Generator().manual_seed(0)
units = torch.randint(0, vc.num_embeddings, (B, U), generator=g)
# deduplicated: no unit equals its predecessor
for t in range(1, U):
    same = units[:, t] == units[:, t - 1]
    units[same, t] = (units[same, t] + 1) % vc.num_embeddings
units = units.to(dev)
langs = [i % vc.num_langs for i in range(B)]
spkrs = [(7 * i) % vc.num_spkrs for i in range(B)]

_, _, dur = eng.resynthesize(units, langs, spkrs)
dur_h = dur.cpu().long()
tot = dur_h.sum(1)
expanded = torch.stack([torch.cat([units[b].cpu().repeat_interleave(dur_h[b]),
                                   units[b, -1:].cpu().repeat(int(tot.max() - tot[b]))]) for b in range(B)]).to(dev)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


expand_ms, gen_ms, plain_ms = [], [], []
with torch.inference_mode():
    for i in range(args.warmup + args.iters):
        t_exp, (x0, lens, _, _) = timed(lambda: eng._expand(units, langs, spkrs))
        t_gen, _ = timed(lambda: eng._generate(x0, lens))
        t_plain, _ = timed(lambda: eng(expanded, langs, spkrs))
        if i >= args.warmup:
            expand_ms.append(t_exp)
            gen_ms.append(t_gen)
            plain_ms.append(t_plain)
        del x0, lens

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
audio_s = float(tot.sum()) * vc.hop / 16000
med = statistics.median
print(f"card: {card}")
print(f"batch {B} x {U} units, durations mean {dur_h.float().mean():.2f} (min {int(dur_h.min())}, max {int(dur_h.max())}), "
      f"frames per row {int(tot.min())}-{int(tot.max())}, {audio_s:.1f} s of audio per call")
for name, ms in (("predictor + expansion", expand_ms), ("generator (ragged, masked)", gen_ms),
                 ("plain generator, host-expanded", plain_ms)):
    print(f"{name:32s} median {med(ms):8.2f} ms  (min {min(ms):8.2f}, max {max(ms):8.2f}, {len(ms)} calls)")
total = med(expand_ms) + med(gen_ms)
print(f"resynthesis: {total:.1f} ms per call, {audio_s / (total / 1e3):.0f} s of audio per second")
