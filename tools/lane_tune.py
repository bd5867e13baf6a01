"""Decoder-step kernel choices (transposed wgmma or the row-major chain / L2 prefetch) timed with 1 and with
`--lanes` beam searches in flight: under lanes the cheapest choice in SM-slot time wins, not the shortest latency chain.
Usage: python tools/lane_tune.py [--lanes 4]"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = [
    ("base", {}),
    ("chain", dict(decode_gemm_t=False)),
    ("no prefetch", dict(decode_prefetch=False)),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=4)
    a = ap.parse_args()
    import bench
    from seamless_communication_b200 import synthetic as S
    from seamless_communication_b200.parallel import LanePool

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    tr = bench.build_models(device)
    eng = tr.model.engine
    waves = S.make_waveforms(32, bench.SAMPLES, seed=1234).to(device)
    enc, _ = eng.encode_speech(tr.fbank_batch(waves)["seqs"], None)
    prefix = [eng.cfg.text_eos, eng.text_tokenizer.lang_index(bench.TGT_LANG)]
    defaults = {k: getattr(eng, k) for k in ("decode_gemm_t", "decode_prefetch")}
    pool1, poolL = LanePool(device, 1, [eng]), LanePool(device, a.lanes, [eng])
    ref = None
    for name, cfg in CONFIGS:
        for k, v in defaults.items():
            setattr(eng, k, cfg.get(k, v))
        eng._graphs.clear()
        try:
            hyps = eng.beam_search(enc, None, prefix, beam=bench.BEAM, hard_max=bench.HARD_MAX)
            torch.cuda.synchronize()
            ids = [h[0][1] for h in hyps]
            ref = ref or ids
            same = sum(x == y for x, y in zip(ids, ref))
            ms1 = bench.lanes_search_ms(pool1, eng, enc, 1)
            msL = bench.lanes_search_ms(poolL, eng, enc, a.lanes)
            print(f"{name:22s}: 1 search {ms1:7.1f} ms | {a.lanes} searches {msL:7.1f} ms = {msL / a.lanes:6.1f} ms each | "
                  f"best hypotheses equal to base: {same}/32", flush=True)
        except Exception as ex:  # a configuration the kernels refuse
            print(f"{name:22s}: {type(ex).__name__}: {ex}", flush=True)
    pool1.close(); poolL.close()


if __name__ == "__main__":
    main()
