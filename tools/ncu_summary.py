"""Per-kernel ncu summary of one S2ST step and the DRAM traffic of one beam-search step.

On a machine with the GPU and Nsight Compute:
    SB_BENCH_HARD_MAX=14 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,\
sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active --clock-control none --csv \
        --log-file step_metrics.csv python bench.py --profile-only
Anywhere:
    python tools/ncu_summary.py step_metrics.csv --hard-max 14
writes profiles/<tag>_kernels_ncu.txt (one line per kernel: launches, mean / total duration, share of the step, DRAM bytes
per launch, achieved GB/s, tensor-pipe %) and profiles/<tag>_decode_step_dram.json (DRAM bytes per beam-search step).
Per-launch times under ncu are cold-cache and serialised: the SHARES are what to compare."""
import argparse
import collections
import csv
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def short(name):
    name = re.sub(r"\(anonymous namespace\)::|<unnamed>::", "", name)
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"^(sb::|at::native::|at::)+", "", name)
    m = re.match(r"([A-Za-z0-9_]+)(<[^>]*>)?", name)
    return (m.group(1) + (m.group(2) or "")) if m else name[:60]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--hard-max", type=int, required=True, help="hard_max_seq_len of the profiled run (decode steps = it - 1)")
    ap.add_argument("--tag", default="r02")
    a = ap.parse_args()
    rows = []
    with open(a.csv, newline="") as f:
        lines = [l for l in f if not l.startswith("==")]
    rd = csv.DictReader(lines)
    launches = collections.OrderedDict()
    for r in rd:
        if "Metric Name" not in r or not r.get("ID"):
            continue
        k = int(r["ID"])
        d = launches.setdefault(k, {"name": short(r["Kernel Name"])})
        try:
            v = float(r["Metric Value"].replace(",", ""))
        except ValueError:
            continue
        unit = r.get("Metric Unit", "")
        mn = r["Metric Name"]
        if mn == "gpu__time_duration.sum":
            v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(unit, 1e-3)  # -> us
        if mn.startswith("dram__bytes"):
            v *= {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1.0)
        d[mn] = v
    seq = list(launches.values())
    total_us = sum(x.get("gpu__time_duration.sum", 0.0) for x in seq)
    agg = collections.OrderedDict()
    for x in seq:
        g = agg.setdefault(x["name"], dict(n=0, us=0.0, rd=0.0, wr=0.0, tensor=0.0))
        g["n"] += 1
        g["us"] += x.get("gpu__time_duration.sum", 0.0)
        g["rd"] += x.get("dram__bytes_read.sum", 0.0)
        g["wr"] += x.get("dram__bytes_write.sum", 0.0)
        g["tensor"] += x.get("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", 0.0)
    out = [f"# ncu per-kernel summary of one S2ST step (hard_max_seq_len {a.hard_max}); {len(seq)} launches, {total_us / 1e3:.1f} ms serialised",
           f"# {'kernel':44s} {'launches':>8s} {'mean us':>9s} {'total ms':>9s} {'share %':>8s} {'dram MB/launch':>15s} {'GB/s':>8s} {'tensor %':>9s}"]
    for name, g in sorted(agg.items(), key=lambda kv: -kv[1]["us"]):
        mb = (g["rd"] + g["wr"]) / g["n"] / 1e6
        gbs = (g["rd"] + g["wr"]) / (g["us"] * 1e-6) / 1e9 if g["us"] > 0 else 0.0
        out.append(f"  {name:44s} {g['n']:8d} {g['us'] / g['n']:9.1f} {g['us'] / 1e3:9.2f} {100 * g['us'] / total_us:8.1f} {mb:15.2f} {gbs:8.0f} "
                   f"{g['tensor'] / g['n']:9.1f}")
    # the beam search = launches from the first embedding-frontend kernel to the last step-advance kernel
    names = [x["name"] for x in seq]
    first = next((i for i, n in enumerate(names) if n.startswith("embed_kernel")), None)
    last = max((i for i, n in enumerate(names) if n.startswith("step_advance_kernel")), default=None)
    dram = None
    if first is not None and last is not None and last > first:
        steps = a.hard_max - 1
        dec = seq[first:last + 1]
        b = sum(x.get("dram__bytes_read.sum", 0.0) + x.get("dram__bytes_write.sum", 0.0) for x in dec)
        us = sum(x.get("gpu__time_duration.sum", 0.0) for x in dec)
        dram = {"dram_bytes_per_step": b / steps, "launches_per_step": len(dec) / steps, "us_per_step_serialised": us / steps,
                "steps_profiled": steps, "mean_position": steps / 2.0,
                "source": f"profiles/{a.tag}_kernels_ncu.txt (ncu dram__bytes_read.sum + dram__bytes_write.sum over the {len(dec)} "
                          f"launches of a {steps}-step search, per step; K/V reads grow with the position, mean position {steps / 2.0:.0f})"}
        out.append(f"# beam search: {len(dec)} launches over {steps} steps = {len(dec) / steps:.1f} per step, "
                   f"{b / steps / 1e9:.3f} GB DRAM traffic per step, {us / steps / 1e3:.3f} ms per step serialised")
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    open(os.path.join(ROOT, "profiles", f"{a.tag}_kernels_ncu.txt"), "w").write("\n".join(out) + "\n")
    if dram:
        json.dump(dram, open(os.path.join(ROOT, "profiles", f"{a.tag}_decode_step_dram.json"), "w"), indent=1)
    print("\n".join(out[:40]))


if __name__ == "__main__":
    main()
