#!/usr/bin/env python
"""Per-launch time of the six weight products of one decoder layer at the bench's beam-search step shape (160 rows,
seamlessM4T_large: model 1024, FFN 8192), on the row-major launch chain (sb_gemm_splitk at the step's K slices, sb_gemm
for FFN inner) and on the transposed kernel (sb_gemm_decode) at each split count it can take, plus the split-K reduction that follows a residual product.
Each CUDA graph chains launches over 24 different weight tensors, so weights come from HBM as in a step.
Prints the card and its power limit with the numbers."""
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
ap.add_argument("--splits", default="1,2,4,5,8,16", help="split counts tried on the transposed kernel")
args = ap.parse_args()

R, LAYERS, REPS, M, FFN = args.rows, 24, 4, 1024, 8192
dev = "cuda"
SPLITS = [int(s) for s in args.splits.split(",")]
S_QKV, S_ATT, S_FFN = ops.decode_splits(R, M, FFN)


def timed(fn):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for i in range(3):
            fn(i % LAYERS)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REPS):
            for i in range(LAYERS):
                fn(i)
    for _ in range(3):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (20 * REPS * LAYERS)


def product(name, n, k, chain, direct=False):
    a = Seq(1, R, k)
    a.buf.normal_()
    ws = [(torch.randn(n, k, device=dev) * 0.02).half() for _ in range(LAYERS)]
    bias = torch.zeros(n, device=dev)
    out = Seq(1, R, n)
    part = torch.empty(max(SPLITS + [16]) * ops.slice_rows(R), n, dtype=torch.float32, device=dev)
    res = []
    if chain == "tc_direct":
        res.append(("chain tc", timed(lambda i: ops.gemm(a, ws[i], n, bias, act=ops.ACT_RELU, out=out))))
    else:
        res.append((f"chain splitk/{chain}", timed(lambda i: ops.gemm_splitk(a, ws[i], n, chain, part))))
    if direct:
        res.append(("T direct", timed(lambda i: ops.gemm_decode(a, ws[i], n, bias, act=ops.ACT_RELU, out=out))))
    for sp in SPLITS:
        if sp <= k // 64:
            res.append((f"T/{sp}", timed(lambda i, sp=sp: ops.gemm_splitk(a, ws[i], n, sp, part, transposed=True))))
    wbytes = n * k * 2
    cols = " | ".join(f"{lab} {t:6.2f} us ({wbytes / t / 1e6:4.2f} TB/s)" for lab, t in res)
    print(f"{name:<16} {n:5d} x {k:5d} : {cols}", flush=True)


def reduce_ln():
    x, h = Seq(1, R, M), Seq(1, R, M)
    x.buf.normal_()
    part = torch.randn(16 * ops.slice_rows(R), M, device=dev)
    lw, lb, b = torch.ones(M, device=dev), torch.zeros(M, device=dev), torch.zeros(M, device=dev)
    cols = " | ".join(f"splits {sp} {timed(lambda i, sp=sp: ops.splitk_reduce_ln(part, sp, b, x, lw, lb, h)):6.2f} us"
                      for sp in (2, 4, 5, 8, 16))
    print(f"{'splitk_reduce_ln':<16} {R:5d} x {M:5d} : {cols}", flush=True)


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}\nrows {R}, per launch (in-graph, 24 distinct weights); TB/s = weight bytes / time")
product("q|k|v", 3 * M, M, S_QKV)
product("self-attn out", M, M, S_ATT)
product("cross q", M, M, S_ATT)
product("cross out", M, M, S_ATT)
product("FFN inner", FFN, M, "tc_direct", direct=True)
product("FFN out", M, FFN, S_FFN)
reduce_ln()
