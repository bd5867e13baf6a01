"""Do two lanes' decoder-step kernels overlap on the device?  For every kernel kind of a step (decode shape: 160 rows,
M 1024, FFN 8192, vocabulary 256206) a CUDA graph of `--reps` back-to-back launches is timed alone and together with
an identical graph on a second stream (own activations / outputs, shared weights).
ratio = t(both) / t(alone): 1.0 = the second lane is free, 2.0 = the kernels run one after the other."""
import argparse
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--streams", type=int, default=2)
    a = ap.parse_args()
    from seamless_communication_b200 import _lib, ops
    from seamless_communication_b200.ops import ACT_RELU, Seq
    dev = "cuda"
    lib = _lib.load()
    R, M, F, V, H, ML, B, S_ENC, BEAM = 160, 1024, 8192, 256206, 16, 102, 32, 63, 5
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: (torch.randn(*s, device=dev, generator=g) * 0.05).half()  # noqa: E731
    w_qkv, w_1, w_2, emb = rnd(3 * M, M), rnd(F, M), rnd(M, F), rnd(V, M)
    b_f, b_m = torch.zeros(F, device=dev), torch.zeros(M, device=dev)
    ln_w, ln_b = torch.ones(M, device=dev), torch.zeros(M, device=dev)
    SR = ops.slice_rows(R)
    zero_bias = torch.zeros(3 * M, device=dev)

    def lane_buffers():
        d = dict(h=Seq(1, R, M, buf=rnd(R, M)), x=Seq(1, R, M, buf=rnd(R, M)), att=Seq(1, R, M, buf=rnd(R, M)),
                 ffn=Seq(1, R, F, buf=rnd(R, F)), part=torch.zeros((16 * SR, M), dtype=torch.float32, device=dev),
                 part_qkv=torch.zeros((4 * SR, 3 * M), dtype=torch.float32, device=dev),
                 logits=Seq(1, R, V, dtype=torch.float32, buf=torch.empty((R, (V + 7) // 8 * 8), dtype=torch.float32, device=dev)),
                 stats=torch.empty(((V + 127) // 128, R, 2), dtype=torch.float32, device=dev),
                 kc=rnd(ML, R, M), vc=rnd(ML, R, M), anc=torch.arange(R, dtype=torch.int32, device=dev)[:, None].repeat(1, ML).contiguous(),
                 step=torch.full((1,), 50, dtype=torch.int32, device=dev), kv=rnd(B * S_ENC, 2 * M),
                 cand_val=torch.empty((R, 11), dtype=torch.float32, device=dev), cand_idx=torch.empty((R, 11), dtype=torch.int32, device=dev),
                 eos=torch.empty((R,), dtype=torch.float32, device=dev))
        return d

    def kinds(d):
        st = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
        return {
            "qkv  wgmma split 2": lambda: ops.gemm_splitk(d["h"], w_qkv, 3 * M, 2, d["part_qkv"]),
            "ffn1 wgmma direct": lambda: ops.gemm(d["h"], w_1, F, b_f, act=ACT_RELU, out=d["ffn"]),
            "ffn2 wgmma split 8": lambda: ops.gemm_splitk(d["ffn"], w_2, M, 8, d["part"]),
            "reduce + LayerNorm": lambda: ops.splitk_reduce_ln(d["part"], 8, b_m, d["x"], ln_w, ln_b, d["h"]),
            "self attention t=50": lambda: _lib.check(lib.sb_decode_self_attn(
                None, d["part_qkv"].data_ptr(), 2, SR, zero_bias.data_ptr(), d["kc"].data_ptr(), d["vc"].data_ptr(),
                d["anc"].data_ptr(), ML, d["step"].data_ptr(), ML, d["att"].buf.data_ptr(), R, H, st()), "self"),
            "cross attention": lambda: _lib.check(lib.sb_decode_cross_attn(
                None, d["part"].data_ptr(), 8, SR, b_m.data_ptr(), d["kv"].data_ptr(), d["kv"][:, M:].data_ptr(), d["kv"].stride(0), None,
                S_ENC, d["att"].buf.data_ptr(), R, BEAM, H, st()), "cross"),
            "vocabulary projection": lambda: ops.gemm(d["h"], emb, V, None, out=d["logits"], out_f32=True, tile_stats=d["stats"]),
            "top-K from tiles": lambda: _lib.check(lib.sb_logits_topk_tiles(
                d["logits"].buf.data_ptr(), d["logits"].buf.stride(0), d["stats"].data_ptr(), R, V, 0, 3, 1, 0.0, 11, d["cand_val"].data_ptr(),
                d["cand_idx"].data_ptr(), d["eos"].data_ptr(), st()), "topk"),
        }

    lanes = [lane_buffers() for _ in range(a.streams)]
    streams = [torch.cuda.Stream() for _ in range(a.streams)]
    names = list(kinds(lanes[0]).keys())
    print(f"{'kernel':26s} {'alone us':>9s} {'x' + str(a.streams) + ' us':>9s}  ratio   ({a.reps} launches per graph)")
    for name in names:
        graphs = []
        try:
            for d, s in zip(lanes, streams):
                fn = kinds(d)[name]
                with torch.cuda.stream(s):
                    fn()
                    torch.cuda.synchronize()
                    gr = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(gr, stream=s):
                        for _ in range(a.reps):
                            fn()
                graphs.append(gr)
        except Exception as ex:
            print(f"{name:26s} {type(ex).__name__}: {ex}")
            continue

        def run(k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            main = torch.cuda.current_stream()
            best = 1e9
            for _ in range(4):
                torch.cuda.synchronize()
                e0.record()
                for s in streams[:k]:
                    s.wait_event(e0)
                for gr, s in zip(graphs[:k], streams[:k]):
                    with torch.cuda.stream(s):
                        gr.replay()
                for s in streams[:k]:
                    main.wait_stream(s)
                e1.record()
                torch.cuda.synchronize()
                best = min(best, e0.elapsed_time(e1))
            return best * 1e3 / a.reps

        t1, tk = run(1), run(a.streams)
        print(f"{name:26s} {t1:9.2f} {tk:9.2f}  {tk / t1:5.2f}", flush=True)


if __name__ == "__main__":
    main()
