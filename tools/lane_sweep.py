"""Throughput of the S2ST step against the number of batches in flight (parallel.LanePool) on one GPU.
Usage: python tools/lane_sweep.py [--lanes 1,2,3,4,6] [--rounds 3]"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", default="1,2,3,4,6")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import bench
    from seamless_communication_b200 import synthetic as S
    from seamless_communication_b200.inference import SequenceGeneratorOptions
    from seamless_communication_b200.parallel import LanePool

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    tr = bench.build_models(device)
    eng = tr.model.engine
    opts = SequenceGeneratorOptions(beam_size=bench.BEAM, soft_max_seq_len=(1, 200), hard_max_seq_len=bench.HARD_MAX)
    waves = S.make_waveforms(32, bench.SAMPLES, seed=1234).to(device)

    def step():
        return tr.predict(tr.fbank_batch(waves), "s2st", bench.TGT_LANG, text_generation_opts=opts)

    texts0, _ = step()
    torch.cuda.synchronize()
    enc, _ = eng.encode_speech(tr.fbank_batch(waves)["seqs"], None)
    main_stream = torch.cuda.current_stream()
    for L in [int(v) for v in a.lanes.split(",")]:
        pool = LanePool(device, L, [eng])
        t0 = time.time()
        pool.warm(step)
        t_warm = time.time() - t0
        n = L * a.rounds
        for timed in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.time()
            e0.record()
            futs = [pool.submit(i, step) for i in range(n)]
            outs = []
            for f in futs:
                out, done = f.result()
                main_stream.wait_event(done)
                outs.append(out)
            e1.record()
            torch.cuda.synchronize()
            wall = time.time() - t0
        same = all(o[0] == texts0 for o in outs)
        ms = e0.elapsed_time(e1)
        ms_search = bench.lanes_search_ms(pool, eng, enc, L)
        print(f"lanes {L}: {n} steps in {ms:.1f} ms (wall {wall * 1e3:.1f}) = {ms / n:.1f} ms/step, {32 * n / ms * 1e3:.1f} utt/s; "
              f"texts identical to serial: {same}; {L} searches alone: {ms_search:.1f} ms; warm {t_warm:.1f}s; "
              f"mem {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB", flush=True)
        pool.close()


if __name__ == "__main__":
    main()
