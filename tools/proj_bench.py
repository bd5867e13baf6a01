#!/usr/bin/env python
"""Time the tied vocabulary projection of one beam-search step (sb_gemm with tile_stats: R rows x 1024 against the
256102 x 1024 embedding, fp32 logits) on the weight-stationary kernel and on the general kernel (SB_PROJ_T=0), with CUDA
events over many launches, alternating the two.  Bytes: the embedding once + h + the fp32 logits + the statistics."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import ops  # noqa: E402
from seamless_communication_b200.ops import Seq  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=160)
ap.add_argument("--vocab", type=int, default=256102)
ap.add_argument("--iters", type=int, default=200)
ap.add_argument("--rounds", type=int, default=3)
args = ap.parse_args()

R, V, K = args.rows, args.vocab, 1024
dev = "cuda"
torch.manual_seed(0)
a = Seq(1, R, K, buf=torch.randn(R, K, device=dev).half())
w = (torch.randn(V, K, device=dev) * 0.05).half()
ld = (V + 7) // 8 * 8
logits = Seq(1, R, V, dtype=torch.float32, buf=torch.empty((R, ld), device=dev))
stats = torch.empty(((V + 127) // 128, R, 2), device=dev)
nbytes = V * K * 2 + R * K * 2 + R * V * 4 + stats.numel() * 4
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}; R={R} V={V} K={K}; {nbytes / 1e6:.1f} MB per call")


def run(proj_t):
    os.environ["SB_PROJ_T"] = proj_t
    for _ in range(10):
        ops.gemm(a, w, V, None, out=logits, out_f32=True, tile_stats=stats)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.iters):
        ops.gemm(a, w, V, None, out=logits, out_f32=True, tile_stats=stats)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / args.iters


for rnd in range(args.rounds):
    for name, flag in (("general (SB_PROJ_T=0)", "0"), ("weight-stationary", "1")):
        us = run(flag)
        gbs = nbytes / (us * 1e-6) / 1e9
        print(f"round {rnd}: {name:22s} {us:8.1f} us  {gbs:7.0f} GB/s  {100 * gbs / 3350:5.1f} % of 3.35 TB/s")
