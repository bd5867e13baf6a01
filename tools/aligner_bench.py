#!/usr/bin/env python
"""Forced-aligner throughput: N rows of U units and ~C characters through synthetic nar_t2u_aligner weights, on the CUDA
path and on a PyTorch fp16 eager arm with the reference's semantics (models/aligner/model.py:146-277: F.conv1d, the
broadcast difference + torch.norm + log_softmax on the device, then the alignment search row by row on the host as a
double loop over numpy scalars), alternated call by call.  The eager arm zeroes padded embeddings, so that both arms
define a ragged row as the row alone and their durations can be compared.

Prints CUDA-event medians of the CUDA path's device stages (embeddings + convs, sb_align_lprob, sb_monotonic_align; the
first event is recorded once the ids are on the device), the wall time of a whole call including its host-side id
checks and copies, the eager arm's device part and host search, duration agreement between the arms, and the card's
name and power limit read in the same run.

  python tools/aligner_bench.py --batch 32 --units 500 --chars 150 --iters 20
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from seamless_communication_b200 import config as C, synthetic as S  # noqa: E402
from seamless_communication_b200.aligner_engine import AlignerEngine  # noqa: E402

STAGES = ["embed + convs", "sb_align_lprob", "sb_monotonic_align"]


def host_search(lp: np.ndarray) -> np.ndarray:
    """Durations of one row by the alignment search as the reference runs it on the host: Python loops over numpy scalars
    (float32 inputs, float64 scores, the first score row as numpy's float32 prefix sums; the loop form of
    tests/oracle_aligner.mas_q with numpy_row0), then the walk back from the last character, counting frames per
    character."""
    n_frames, n_chars = lp.shape
    score = np.full((n_chars, n_frames), -np.inf)
    for col in range(n_frames):
        score[0, col] = np.sum(lp[:col + 1, 0])
    for col in range(1, n_frames):
        for row in range(1, min(col, n_chars - 1) + 1):
            stay, advance = score[row, col - 1], score[row - 1, col - 1]
            score[row, col] = (advance if advance >= stay else stay) + lp[col, row]
    counts = np.zeros(n_chars, dtype=np.int64)
    row = n_chars - 1
    counts[row] += 1
    for col in range(n_frames - 2, -1, -1):
        if row > 0 and score[row - 1, col] >= score[row, col]:
            row -= 1
        counts[row] += 1
    return counts


class Eager:
    def __init__(self, cfg, sd, dev):
        self.cfg = cfg
        self.sd = {k: v.to(dev, torch.float16) for k, v in sd.items()}

    def _convs(self, x, prefix, n):
        h = x.transpose(1, 2)
        for i in range(n):
            w, b = self.sd[f"{prefix}.{1 + 3 * i}.weight"], self.sd[f"{prefix}.{1 + 3 * i}.bias"]
            h = F.conv1d(h, w, b, padding=w.shape[2] // 2)
            if i < n - 1:
                h = F.relu(h)
        return h.transpose(1, 2)

    @torch.inference_mode()
    def device_part(self, tids, uids, tl, ul):
        cfg, sd = self.cfg, self.sd
        tmask = (torch.arange(tids.shape[1], device=tids.device)[None] < tl[:, None])
        umask = (torch.arange(uids.shape[1], device=uids.device)[None] < ul[:, None])
        te = sd["alignment_frontend.embed_text.weight"][tids] * tmask[..., None]
        ue = sd["alignment_frontend.embed_unit.weight"][uids] * umask[..., None]
        t = self._convs(te, "alignment_encoder.t_conv", cfg.num_text_layers)
        f = self._convs(ue, "alignment_encoder.f_conv", cfg.num_feat_layers)
        dist = torch.norm(f.unsqueeze(2) - t.unsqueeze(1), p=2, dim=3)
        score = (-cfg.temperature * dist).masked_fill(~tmask[:, None, :], -np.inf)
        return F.log_softmax(score, dim=-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--units", type=int, default=500)
    ap.add_argument("--chars", type=int, default=150)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--arch", default="nar_t2u_aligner")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("aligner_bench.py measures the GPU; no CUDA device is present")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    cfg = C.ALIGNER_ARCHS[a.arch]()
    sd = S.make_aligner_state_dict(cfg, seed=4)
    eng = AlignerEngine(cfg, sd)
    eager = Eager(cfg, sd, "cuda")
    g = torch.Generator().manual_seed(0)
    tl = [a.chars - 10 + int(x) for x in torch.randint(0, 21, (a.batch,), generator=g)]
    ul = [a.units] * a.batch
    tids = torch.randint(4, 40, (a.batch, max(tl)), generator=g)
    uids = torch.randint(4, cfg.num_units + 4, (a.batch, a.units), generator=g)
    for b, n in enumerate(tl):
        tids[b, n:] = cfg.unit_pad_idx
    tids_d, uids_d = tids.cuda(), uids.cuda()
    tl_d, ul_d = torch.tensor(tl).cuda(), torch.tensor(ul).cuda()
    times = {s: [] for s in STAGES}
    total, wall, eager_dev, eager_host, agree = [], [], [], [], []
    for it in range(a.warmup + a.iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        _, dur = eng.forward(tids, uids, tl, ul, marks=ev)
        torch.cuda.synchronize()
        w1 = time.perf_counter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lp = eager.device_part(tids_d, uids_d, tl_d, ul_d)
        e1.record()
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        lp_h = lp.float().cpu().numpy()
        ref = [host_search(lp_h[b, :ul[b], :tl[b]]) for b in range(a.batch)]
        h1 = time.perf_counter()
        if it < a.warmup:
            continue
        for i, s in enumerate(STAGES):
            times[s].append(ev[i].elapsed_time(ev[i + 1]))
        total.append(ev[0].elapsed_time(ev[3]))
        wall.append((w1 - w0) * 1e3)
        eager_dev.append(e0.elapsed_time(e1))
        eager_host.append((h1 - h0) * 1e3)
        d = dur.cpu().numpy()
        agree.append(sum(int(d[b, :tl[b]].tolist() == ref[b].tolist()) for b in range(a.batch)) / a.batch)
    print(f"{gpu}; {a.batch} rows x {a.units} units x {min(tl)}-{max(tl)} characters, {a.arch}; medians of {a.iters}")
    for s in STAGES:
        print(f"{s:<22}{statistics.median(times[s]):9.3f} ms")
    tm, ed, eh = statistics.median(total), statistics.median(eager_dev), statistics.median(eager_host)
    tw = statistics.median(wall)
    print(f"{'CUDA path, device':<22}{tm:9.3f} ms")
    print(f"{'CUDA path, whole call':<22}{tw:9.3f} ms  (wall clock, with the host-side id checks and copies)")
    print(f"{'eager device part':<22}{ed:9.3f} ms  (embeddings, convs, difference tensor + norm, log_softmax)")
    print(f"{'eager host search':<22}{eh:9.3f} ms  (copy to host + the per-row search)")
    print(f"rows whose durations agree between the arms: {100 * statistics.mean(agree):.1f} %")
    print(json.dumps({"gpu": gpu, "batch": a.batch, "units": a.units, "chars": [min(tl), max(tl)], "arch": a.arch,
                      "stage_ms": {s: statistics.median(times[s]) for s in STAGES}, "device_ms": tm, "call_ms": tw,
                      "eager_device_ms": ed, "eager_host_ms": eh, "duration_row_agreement": statistics.mean(agree)}))


if __name__ == "__main__":
    main()
