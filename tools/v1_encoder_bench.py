#!/usr/bin/env python
"""Time the w2v-BERT v1 speech encoder (seamlessM4T_large, arch `base`) against the v2 encoder (`base_v2`) on a batch of
10 s utterances (default 32 x 160000 samples -> 499 frames after the stride-2 frontend), and the two fused attention
modes alone at the same shape:
  * encoder: UnitYEngine.encode_speech (24 Conformer layers + adaptor) on device fbank;
  * attention: one layer's sb_attention_relpos (Transformer-XL: q+u against K, q+v against the staged R window) and
    sb_attention with the Shaw table (64 left, 8 right), on the same q/k/v;
  * the v1 layer's R = r_proj(pos table) GEMM alone.
Times are CUDA-event medians over --iters calls after --warmup calls.  The algorithmic FLOP count of each piece is
printed next to it (QK^T and PV: 4 S^2 64 per head; the Transformer-XL term adds 2 S (2S-1) 64 per head as the
reference computes it; R: 2 (2S-1) M^2).  Also prints the card's name and power limit."""
import argparse
import dataclasses
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import config as C, ops, synthetic as S  # noqa: E402
from seamless_communication_b200.engine import UnitYEngine  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--samples", type=int, default=160000)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
args = ap.parse_args()
dev = "cuda"


def timed(fn):
    ms = []
    for i in range(args.warmup + args.iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            ms.append(e0.elapsed_time(e1))
    return statistics.median(ms), min(ms), max(ms)


def report(name, t, flop):
    med, lo, hi = t
    print(f"{name:34s} median {med:8.3f} ms (min {lo:8.3f}, max {hi:8.3f})  {flop / 1e9:9.1f} GFLOP  {flop / med / 1e9:7.1f} TFLOP/s")


card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print(f"card: {card}")
B = args.batch
waves = S.make_waveforms(B, args.samples, seed=5).to(dev)
T_fb = 1 + (args.samples - 400) // 160
fb, frames = ops.fbank(waves, torch.full((B,), args.samples, dtype=torch.int32, device=dev), T_fb + T_fb % 2)
S_ = fb.shape[1] // 2
M, H, L, F_ = 1024, 16, 24, 4096
# encoder FLOP per layer (GEMMs): 2 FFNs, q|k|v, out, pointwise convs; attention; v1 adds R and the positional scores
gemm = 2 * B * S_ * (2 * 2 * M * F_ + 3 * M * M + M * M + 2 * M * M + M * M)
attn_plain = 4 * B * H * S_ * S_ * 64
attn_xl = attn_plain + 2 * B * H * S_ * (2 * S_ - 1) * 64
r_gemm = 2 * (2 * S_ - 1) * M * M
print(f"batch {B} x {args.samples} samples -> {S_} frames")
with torch.inference_mode():
    for arch in ("base", "base_v2"):
        # only the encoder runs: a one-layer decoder with a small vocabulary keeps the synthetic weights small
        cfg = dataclasses.replace(C.UNITY_ARCHS[arch](), dec_layers=1, text_vocab=8192 + 102)
        eng = UnitYEngine(cfg, S.make_unity_state_dict(cfg, 0, with_t2u=False), S.make_tokenizers(cfg))
        flop = L * (gemm + (attn_xl + r_gemm if arch == "base" else attn_plain))
        report(f"encoder {arch} ({cfg.encoder_variant})", timed(lambda: eng.encode_speech(fb, frames)), flop)
        if arch == "base":
            pos = ops.Seq(1, 2 * S_ - 1, M, buf=eng.w["relpos"][4096 - S_:4096 + S_ - 1])
            wr = eng.w["speech_encoder.inner.layers.0.r_proj.w"]
            report("R = r_proj(pos) GEMM", timed(lambda: ops.gemm(pos, wr, M)), r_gemm)
        del eng
        torch.cuda.empty_cache()
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = ops.Seq(B, S_, 3 * M, buf=torch.randn(B * S_, 3 * M, device=dev, generator=g).half(),
                  lens=torch.full((B,), S_, dtype=torch.int32, device=dev))
    r = torch.randn(2 * S_ - 1, M, device=dev, generator=g).half()
    vb = torch.randn(H, 64, device=dev, generator=g)
    rel_k = torch.randn(73, 64, device=dev, generator=g).half()
    report("attention Transformer-XL (v1)", timed(lambda: ops.self_attention_relpos(qkv, H, r, vb=vb)), attn_xl)
    report("attention Shaw (v2)", timed(lambda: ops.self_attention(qkv, H, rel_k=rel_k, rel_left=64, rel_right=8)), attn_plain)
