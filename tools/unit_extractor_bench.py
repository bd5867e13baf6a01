#!/usr/bin/env python
"""Unit extractor throughput: N x S s of synthetic audio through xlsr2_1b_v2 up to one layer and a K-centroid codebook,
on the CUDA path and on a PyTorch fp16 eager arm over the same weights (F.conv1d, F.layer_norm, F.gelu,
F.scaled_dot_product_attention, matmul + argmin), alternated call by call.

Prints CUDA-event medians per stage (front, conv stack, projection + positional conv, encoder layers, k-means), the
algorithmic FLOPs of each stage computed from the shapes below and its share of the H100 SXM's 989 TFLOP/s dense fp16
data-sheet rate, utterances per second of both arms, their unit agreement, and the card's name and power limit read in
the same run.  Synthetic weights are drawn for the layers that run only (the engine never reads the others).

  python tools/unit_extractor_bench.py --batch 32 --seconds 10 --layer 34 --centroids 10000 --iters 5
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from seamless_communication_b200 import config as C, synthetic as S  # noqa: E402
from seamless_communication_b200.wav2vec2_engine import Wav2Vec2Engine, conv_frames  # noqa: E402

PEAK = 989e12
STAGES = ["front", "conv stack", "proj + pos conv", "layers", "k-means"]


def stage_flops(cfg, B, L, layers, K):
    d = cfg.feature_extractor_layer_descs
    fr = conv_frames(L, d)
    M, Fd = cfg.model_dim, cfg.ffn_inner_dim
    T = fr[-1]
    conv = sum(2 * B * fr[i] * c * d[i - 1][0] * k for i, (c, k, _) in enumerate(d) if i > 0)
    proj = 2 * B * T * 512 * M + 2 * B * T * M * (M // cfg.num_pos_conv_groups) * cfg.pos_conv_kernel_size
    layer = 2 * B * T * M * (3 * M + M + 2 * Fd) + 4 * B * T * T * M
    return [2 * B * fr[0] * 512 * 10, conv, proj, layers * layer, 2 * B * T * M * K]


class Eager:
    """The same computation in PyTorch fp16 on the device (batch padded; masks as the reference applies them)."""

    def __init__(self, cfg, sd, centroids, layers, dev):
        h = lambda t: t.to(dev, torch.float16)  # noqa: E731
        self.cfg, self.layers = cfg, layers
        self.sd = {k: h(v) for k, v in sd.items() if not k.startswith("encoder.layers.") or int(k.split(".")[2]) < layers}
        p = "encoder_frontend.pos_encoder.conv"
        v, g = sd[p + ".weight_v"].double(), sd[p + ".weight_g"].double().reshape(-1)
        self.pos_w = h(v * (g / v.pow(2).sum((0, 1)).sqrt())[None, None, :])
        self.c = h(centroids)
        self.cn = self.c.float().pow(2).sum(1)

    @torch.inference_mode()
    def __call__(self, wave, lens):
        sd, cfg = self.sd, self.cfg
        B = wave.shape[0]
        Lp = [n + n % 2 for n in lens]
        x = torch.zeros(B, max(Lp), device=wave.device)
        for b, n in enumerate(lens):
            x[b, :n] = wave[b, :n]
            if n % 2:
                x[b, n] = 1.0
            r = x[b, :Lp[b]]
            x[b, :Lp[b]] = (r - r.mean()) / torch.sqrt(r.var(unbiased=False) + 1e-5)
        h = x.half()[:, None]
        for i, (c, k, s) in enumerate(cfg.feature_extractor_layer_descs):
            p = f"encoder_frontend.feature_extractor.layers.{i}"
            h = F.conv1d(h, sd[p + ".conv.weight"], sd[p + ".conv.bias"], stride=s)
            h = F.gelu(F.layer_norm(h.transpose(1, 2), (c,), sd[p + ".layer_norm.weight"], sd[p + ".layer_norm.bias"]).transpose(1, 2))
        h = h.transpose(1, 2)
        h = F.layer_norm(h, (512,), sd["encoder_frontend.post_extract_layer_norm.weight"], sd["encoder_frontend.post_extract_layer_norm.bias"])
        h = F.linear(h, sd["encoder_frontend.model_dim_proj.weight"], sd["encoder_frontend.model_dim_proj.bias"])
        mask = [conv_frames(n, cfg.feature_extractor_layer_descs)[-1] for n in lens]
        T = h.shape[1]
        keep = torch.arange(T, device=h.device)[None] < torch.tensor(mask, device=h.device)[:, None]
        h = h * keep[..., None]
        y = F.conv1d(h.transpose(1, 2), self.pos_w, sd["encoder_frontend.pos_encoder.conv.bias"], padding=64,
                     groups=cfg.num_pos_conv_groups)[:, :, :-1]
        h = h + F.gelu(y.transpose(1, 2))
        H, M = cfg.num_encoder_attn_heads, cfg.model_dim
        am = keep[:, None, None, :]
        for i in range(self.layers):
            p = f"encoder.layers.{i}"
            a = F.layer_norm(h, (M,), sd[p + ".self_attn_layer_norm.weight"], sd[p + ".self_attn_layer_norm.bias"])
            q, k, v = (F.linear(a, sd[f"{p}.self_attn.{n}_proj.weight"], sd[f"{p}.self_attn.{n}_proj.bias"])
                       .view(B, T, H, M // H).transpose(1, 2) for n in "qkv")
            a = F.scaled_dot_product_attention(q, k, v, attn_mask=am).transpose(1, 2).reshape(B, T, M)
            h = h + F.linear(a, sd[p + ".self_attn.output_proj.weight"], sd[p + ".self_attn.output_proj.bias"])
            a = F.layer_norm(h, (M,), sd[p + ".ffn_layer_norm.weight"], sd[p + ".ffn_layer_norm.bias"])
            h = h + F.linear(F.gelu(F.linear(a, sd[p + ".ffn.inner_proj.weight"], sd[p + ".ffn.inner_proj.bias"])),
                             sd[p + ".ffn.output_proj.weight"], sd[p + ".ffn.output_proj.bias"])
        d = self.cn[None, None] - 2 * (h @ self.c.t()).float()
        u = d.argmin(-1)
        return [u[b, :conv_frames(Lp[b], cfg.feature_extractor_layer_descs)[-1]] for b in range(B)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--layer", type=int, default=34)
    ap.add_argument("--centroids", type=int, default=10000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--arch", default="xlsr2_1b_v2")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("unit_extractor_bench.py measures the GPU; no CUDA device is present")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cfg = C.WAV2VEC2_ARCHS[a.arch]()
    cfg.num_encoder_layers = a.layer + 1  # only layers 0..layer run
    sd = S.make_wav2vec2_state_dict(cfg, seed=3)
    cent = S.make_kmeans_centroids(a.centroids, cfg.model_dim, seed=4, scale=0.5)
    eng = Wav2Vec2Engine(cfg, sd, cent, device="cuda")
    eager = Eager(cfg, sd, cent, a.layer + 1, "cuda")
    L = int(a.seconds * 16000)
    wave = (0.1 * torch.randn(a.batch, L, generator=torch.Generator().manual_seed(0))).cuda()
    lens = [L] * a.batch
    times = {s: [] for s in STAGES}
    total, eager_t = [], []
    for it in range(a.warmup + a.iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        ev[5].record()
        feats, n_out = eng.forward(wave, lens, a.layer, marks=ev)
        units = eng.units(feats, n_out)
        ev[4].record()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ref = eager(wave, lens)
        e1.record()
        torch.cuda.synchronize()
        if it < a.warmup:
            continue
        marks = [ev[5]] + ev[:5]
        for i, s in enumerate(STAGES):
            times[s].append(marks[i].elapsed_time(marks[i + 1]))
        total.append(ev[5].elapsed_time(ev[4]))
        eager_t.append(e0.elapsed_time(e1))
    agree = sum(int((u == r).sum()) for u, r in zip(units, ref)) / sum(len(u) for u in units)
    fl = stage_flops(cfg, a.batch, L, a.layer + 1, a.centroids)
    print(f"{gpu}; {a.batch} x {a.seconds:g} s, {a.arch} layer {a.layer}, {a.centroids} centroids; medians of {a.iters}")
    print(f"{'stage':<18}{'ms':>9}{'GFLOP':>10}{'TFLOP/s':>9}{'of 989':>8}")
    for s, f in zip(STAGES, fl):
        ms = statistics.median(times[s])
        print(f"{s:<18}{ms:9.2f}{f / 1e9:10.1f}{f / ms / 1e9:9.1f}{100 * f / ms / 1e9 / 989:7.1f}%")
    tm, te = statistics.median(total), statistics.median(eager_t)
    print(f"{'total':<18}{tm:9.2f}{sum(fl) / 1e9:10.1f}{sum(fl) / tm / 1e9:9.1f}{100 * sum(fl) / tm / 1e9 / 989:7.1f}%")
    print(f"CUDA path {a.batch / tm * 1e3:.1f} utt/s, PyTorch fp16 eager {a.batch / te * 1e3:.1f} utt/s ({te:.2f} ms); "
          f"unit agreement {100 * agree:.2f} %")
    print(json.dumps({"gpu": gpu, "batch": a.batch, "seconds": a.seconds, "layer": a.layer, "centroids": a.centroids,
                      "stage_ms": {s: statistics.median(times[s]) for s in STAGES}, "total_ms": tm, "eager_ms": te,
                      "utt_per_s": a.batch / tm * 1e3, "eager_utt_per_s": a.batch / te * 1e3, "unit_agreement": agree,
                      "stage_gflop": dict(zip(STAGES, [f / 1e9 for f in fl]))}))


if __name__ == "__main__":
    main()
