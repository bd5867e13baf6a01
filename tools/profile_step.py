#!/usr/bin/env python
"""Kernel-time breakdown of one bench step (one s2st batch through the whole path) with torch.profiler; CUPTI sees the
ctypes-launched kernels too.  Prints the card, its power limit and the table; --out also writes them to a file."""
import argparse
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from seamless_communication_b200 import synthetic as S  # noqa: E402
from seamless_communication_b200.inference import SequenceGeneratorOptions  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None, help="also write the breakdown to this file")
ap.add_argument("--rows", type=int, default=40, help="kernels listed")
args = ap.parse_args()

dev = torch.device("cuda", 0)
cfg = bench.CONFIGS["s2st"]
tr = bench.build_models(dev)
opts = SequenceGeneratorOptions(beam_size=bench.BEAM, soft_max_seq_len=(1, 200), hard_max_seq_len=bench.HARD_MAX)
waves = S.make_waveforms(cfg["batch"], bench.SAMPLES, seed=1234).to(dev)
for _ in range(2):
    tr.predict(tr.fbank_batch(waves), cfg["task"], bench.TGT_LANG, text_generation_opts=opts)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    tr.predict(tr.fbank_batch(waves), cfg["task"], bench.TGT_LANG, text_generation_opts=opts)
    torch.cuda.synchronize()
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
env = " ".join(f"{k}={v}" for k, v in sorted(os.environ.items()) if k.startswith("SB_"))
head = f"card: {card}\nworkload: {cfg['workload']}\nenv: {env or '(defaults)'}\n"
tab = prof.key_averages().table(sort_by="cuda_time_total", row_limit=args.rows, max_name_column_width=90)
print(head + tab)
if args.out:
    with open(args.out, "w") as f:
        f.write(head + tab)
