"""In-graph time per launch of the decoder-step GEMMs (160 rows): wgmma split-K kernel vs the mma.sync skinny kernel.
Each graph chains 96 launches over 24 different weight tensors (a decoder step never re-reads a weight from L2)."""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import ops
from seamless_communication_b200.ops import Seq

R, LAYERS, REPS = 160, 24, 4
dev = "cuda"


def bench(name, n, k, variants):
    a = Seq(1, R, k); a.buf.normal_()
    ws = [(torch.randn(n, k, device=dev) * 0.02).half() for _ in range(LAYERS)]
    bias = torch.zeros(n, device=dev)
    out = Seq(1, R, n)
    part = torch.empty(32 * ops.slice_rows(R), n, dtype=torch.float32, device=dev)
    res = []
    for label, fn in variants(a, ws, bias, out, part):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for i in range(3):
                fn(i % LAYERS)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for r in range(REPS):
                for i in range(LAYERS):
                    fn(i)
        for _ in range(3):
            g.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            g.replay()
        e1.record(); torch.cuda.synchronize()
        res.append("%s %.2f us" % (label, e0.elapsed_time(e1) * 1e3 / (10 * REPS * LAYERS)))
    print("%-28s N=%5d K=%5d : %s" % (name, n, k, " | ".join(res)), flush=True)


def splitk_variants(splits_tc, splits_sk):
    def v(a, ws, bias, out, part):
        for sp in splits_tc:
            yield "tc/%d" % sp, (lambda i, sp=sp: ops.gemm_splitk(a, ws[i], ws[i].shape[0], sp, part))
        for sp in splits_sk:
            yield "sk/%d" % sp, (lambda i, sp=sp: ops.gemm_splitk(a, ws[i], ws[i].shape[0], sp, part, skinny=True))
    return v


def direct_variants(a, ws, bias, out, part):
    yield "tc", (lambda i: ops.gemm(a, ws[i], ws[i].shape[0], bias, act=ops.ACT_RELU, out=out))
    yield "sk", (lambda i: ops.gemm_skinny(a, ws[i], ws[i].shape[0], bias, act=ops.ACT_RELU, out=out))


bench("qkv", 3072, 1024, splitk_variants([2], [1, 2, 4, 8]))
bench("attn out / q proj", 1024, 1024, splitk_variants([4], [2, 4, 8, 16]))
bench("ffn inner (bias+relu, fp16)", 8192, 1024, direct_variants)
bench("ffn inner split", 8192, 1024, splitk_variants([], [1, 2]))
bench("ffn out", 1024, 8192, splitk_variants([8], [8, 16, 32]))
