"""Many concurrent SeamlessStreaming streams: StreamingS2STBatch against N independent StreamingS2ST objects fed the same
ticks, alternating in one process.  N seeded synthetic streams of different lengths and start ticks, 320 ms segments.
Reports per tick: device time (CUDA events), launches, and host syncs (counted by torch's sync debug mode, the same way
for both arms: in the whole tick and in its policy stage); per stream: the real-time factor (device time of the ticks the
stream took part in / its audio).  The first repetition counts syncs and compares the two arms' outputs (text ids, units,
waveform chunks per tick and stream); the last one is timed without sync counting.  Prints the card and its power limit
beside the numbers.

    python tools/streaming_batch_bench.py --streams 1 8 32 64 --arch large
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings
from contextlib import contextmanager, nullcontext

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from seamless_communication_b200 import config as C, ops, synthetic as S  # noqa: E402
from seamless_communication_b200.models.monotonic_decoder import load_monotonic_decoder_model  # noqa: E402
from seamless_communication_b200.models.unity import load_unity_model  # noqa: E402
from seamless_communication_b200.models.vocoder import load_vocoder_model  # noqa: E402
from seamless_communication_b200.streaming import StreamingS2STBatch  # noqa: E402
from seamless_communication_b200.streaming.pipeline import StreamingS2ST  # noqa: E402

SEG = 5120  # 320 ms at 16 kHz


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def models(arch):
    if arch == "tiny":
        cfg, vc, ua, va, ma = C.tiny_v2(), C.tiny_vocoder(), "tiny_v2", "tiny", "tiny_v2"
    else:
        cfg, vc, ua, va, ma = C.base_v2(), C.base_vocoder(), "seamlessM4T_v2_large", "vocoder_v2", "base_v2"
    toks = S.make_tokenizers(cfg)
    unity = load_unity_model(ua, state_dict=S.make_unity_state_dict(cfg, seed=0, dec_gain=4.0), tokenizers=toks)
    voc = load_vocoder_model(va, state_dict=S.make_vocoder_state_dict(vc, seed=1))
    mono = load_monotonic_decoder_model(ma, state_dict=S.make_monotonic_state_dict(cfg, seed=2), tokenizers=toks)
    return unity, mono, voc


def schedule(n, max_segments, seed):
    """(start tick, segments) per stream: lengths in [max/2, max], starts in [0, max/2)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(max(1, max_segments // 2), max_segments + 1, (n,), generator=g).tolist()
    starts = torch.randint(0, max(1, max_segments // 2), (n,), generator=g).tolist()
    waves = S.make_waveforms(n, max_segments * SEG, seed=seed)
    return [(s, [waves[i, k * SEG:(k + 1) * SEG] for k in range(l)]) for i, (s, l) in enumerate(zip(starts, lens))]


class SyncCounter:
    """Host syncs inside `with counter.on():` blocks, counted by torch.cuda's sync debug mode."""

    def __init__(self):
        self.n = 0

    @contextmanager
    def on(self):
        prev = torch.cuda.get_sync_debug_mode()  # blocks nest: the policy stage inside a tick
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                yield
            finally:
                torch.cuda.set_sync_debug_mode(prev)
        self.n += sum("called a synchronizing CUDA operation" in str(w.message) for w in caught)


def counted(fn, counter):
    def wrapped(*a, **k):
        with counter.on():
            return fn(*a, **k)
    return wrapped


def run(kind, unity, mono, voc, sched, lang, opts, count):
    """All ticks of the schedule; returns per-tick (device ms, launches, syncs in the tick, syncs in its policy stage),
    per-stream RTF and per-stream outputs.  Syncs are counted only when `count` (the counting slows the host)."""
    n_ticks = max(s + len(segs) for s, segs in sched)
    if kind == "batch":
        drv = StreamingS2STBatch(unity, mono, voc)
        ids = [drv.add_stream(lang, **opts) for _ in sched]
    else:
        alone = [StreamingS2ST(unity, mono, voc, lang, **opts) for _ in sched]
    pol = SyncCounter()
    if count:
        if kind == "batch":
            drv._policy = counted(drv._policy, pol)
        else:
            for st in alone:
                st.policy.policy = counted(st.policy.policy, pol)
    ticks, busy, outputs = [], [0.0] * len(sched), [[] for _ in sched]
    for t in range(n_ticks):
        live = [i for i, (s, segs) in enumerate(sched) if s <= t < s + len(segs)]
        if not live:
            continue
        torch.cuda.synchronize()
        n0, p0 = ops.launch_count(), pol.n
        tick = SyncCounter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        with tick.on() if count else nullcontext():
            if kind == "batch":
                res = drv.push({ids[i]: sched[i][1][t - sched[i][0]] for i in live},
                               finished={ids[i] for i in live if t - sched[i][0] == len(sched[i][1]) - 1})
                res = [res[ids[i]] for i in live]
            else:
                res = []
                for i in live:
                    k = t - sched[i][0]
                    res.append(alone[i].push(sched[i][1][k], finished=k == len(sched[i][1]) - 1))
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        ticks.append((ms, ops.launch_count() - n0, tick.n + pol.n - p0, pol.n - p0))
        for i, r in zip(live, res):
            outputs[i].append(r)
        for i in live:
            busy[i] += ms
    rtf = [busy[i] * 1e-3 / (len(segs) * 0.32) for i, (_, segs) in enumerate(sched)]
    return ticks, rtf, outputs


def compare(a, b):
    """Ticks (over all streams) whose text ids, units or waveform differ between the arms; the largest waveform difference."""
    differ, err = 0, 0.0
    for sa, sb in zip(a, b):
        for (n1, u1, w1), (n2, u2, w2) in zip(sa, sb):
            same = n1 == n2 and (u1 is None) == (u2 is None) and (u1 is None or torch.equal(u1, u2))
            same = same and (w1 is None) == (w2 is None)
            if same and w1 is not None:
                if w1.shape != w2.shape:
                    same = False
                else:
                    err = max(err, (w1.float() - w2.float()).abs().max().item())
            differ += not same
    return differ, err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 8, 32, 64])
    ap.add_argument("--segments", type=int, default=16, help="longest stream, in 320 ms segments")
    ap.add_argument("--arch", choices=["large", "tiny"], default="large")
    ap.add_argument("--reps", type=int, default=2, help="alternating repetitions of both arms (the first counts syncs and "
                    "compares outputs; the last is timed)")
    args = ap.parse_args()
    name, power = card()
    unity, mono, voc = models(args.arch)
    opts = dict(max_len_b=40)
    print(json.dumps({"card": name, "power_limit": power, "arch": args.arch, "segment_ms": 320}))
    for n in args.streams:
        sched = schedule(n, args.segments, seed=n)
        res, syncs, outs = {}, {}, {}
        for rep in range(max(2, args.reps)):
            for kind in ("batch", "alone"):
                ticks, rtf, out = run(kind, unity, mono, voc, sched, "spa", opts, count=rep == 0)
                if rep == 0:
                    syncs[kind], outs[kind] = ticks, out
                else:
                    res[kind] = (ticks, rtf)
        differ, err = compare(outs["batch"], outs["alone"])
        line = {"streams": n, "card": name, "power_limit": power,
                "outputs": {"ticks_differing": differ, "ticks_compared": sum(len(o) for o in outs["batch"]),
                            "waveform_max_abs_diff": err}}
        for kind, (ticks, rtf) in res.items():
            ms = [x[0] for x in ticks]
            line[kind] = {"ticks": len(ticks), "device_ms_per_tick_mean": statistics.mean(ms), "device_ms_per_tick_max": max(ms),
                          "launches_per_tick": statistics.mean(x[1] for x in ticks),
                          "host_syncs_per_tick": statistics.mean(x[2] for x in syncs[kind]),
                          "policy_host_syncs_per_tick": statistics.mean(x[3] for x in syncs[kind]),
                          "rtf_per_stream_mean": statistics.mean(rtf), "rtf_per_stream_max": max(rtf)}
        print(json.dumps(line))


if __name__ == "__main__":
    main()
