"""sb_gemm (csrc/gemm_tcgen05.cu) through the raw C ABI, against a float64 restatement of its contract
(include/seamless_b200.h, sb_gemm_t), on every tile width, store path and epilogue the host can select.

The contract, field by field, as the reference below computes it:
  acc[m, n] = sum_{tap < taps, c < c_in} A[a_row0 + m + tap*dil, c] * W[n, tap*c_in + c]; rows outside [0, a_rows) read
  as zero and channels c_in..a_ld-1 of a row are never read.  v = act(acc + bias) (GLU: pairs (2j, 2j+1) -> a sigmoid(b)),
  out[q] = gamma (alpha v + res1[q] + res2[q]) with q = m + out_row0, rows whose sequence position (seq_rows / seq_halo /
  seq_len or seq_lens) is outside [0, len) written as 0, out2 = lrelu(out, out2_slope).

Canaries.  Every input element the call must not read is NaN: A rows before the buffer start and at or past a_rows,
columns c_in..a_ld-1, W rows past n, bias past n, residuals on rows outside the output window, on masked rows and past
the output columns.  Every output element outside the written region holds SENT and must survive bit for bit.

Exact family.  a in {-4..4}/4, w in {-4..4}/8: every product is a multiple of 2^-5 of magnitude <= 1/2, so for K up to
10 240 (128 taps x 80) every partial sum is a multiple of 2^-5 below 2^13: at most 2^18 steps, 6 bits short of fp32's
24.  Bias and residuals on a 1/32 grid (magnitude <= 2), alpha, gamma in {0.5, 1, 2}, act in {none, relu, lrelu 2^-3},
out2_slope 2^-3 add at most 4 more bits.  So every fp32 value the kernel forms is the exact value, whatever the
accumulation order, and the check has no tolerance: fp32 outputs equal the float64 reference, fp16 outputs equal
fp16(reference).  This assumes that wgmma sums exactly representable fp16 products exactly; the CUDA-core sb_gemm_ref is
held to the same equality, so a difference confined to sb_gemm would show a hardware rounding, not a contract error.

Bounded family: full-mantissa fp16 inputs, weights scaled so the pre-activation has a standard deviation of about 40
(|x| up to ~150, where __expf saturates), SiLU, GELU, tanh, lrelu 0.1, GLU, out2_slope 0.01 / 0.1.  Per element, with
u = 2^-24 (fp32 unit roundoff) and U_TC = 2^-23 (tensor-core accumulation may truncate instead of round):
  pre-activation  E0 = gamma_{K+2}(U_TC) (sum |a| |w| + |b|),  K = taps * c_in products, the bias add and one spare.
  activation      Ey = L E0 + r(x) (|f(x)| + L E0) + 2^-110 (|x| + E0), L the Lipschitz constant of f and r(x) its
                  relative fp32 error from the CUDA tables (CUDA C++ Programming Guide, intrinsic and single-precision
                  function tables; 1 ulp <= 2^-23 of the value):
                    SiLU  x / (1 + __expf(-x)) via __fdividef: L = 1.1; __expf 2 + floor(1.173 |x|) ulp, __fdividef 2 ulp,
                          the add u: r = (4 + 1.173 (|x| + E0)) 2^-23 + u.
                    GELU  0.5 x (1 + erff(x / sqrt 2)): L = 1.13; erff 2 ulp <= 2^-22 absolute, its argument's rounding
                          (erf' <= 1.13) 1.13 u |x / sqrt 2|, the add 2u absolute, the product u |y|: the bound is written
                          out absolute, 0.5 |x| (2^-22 + 0.8 u |x| + 2u) + u |y|.
                    tanhf 2 ulp: L = 1, r = 2^-22.   lrelu s: L = 1, the product u |s x|.   relu, none: exact.
                    GLU   __fdividef(a, 1 + __expf(-b)): Ea + |a| Eb / 4 + Ea Eb / 4 plus r(b) (|a sigmoid(b)| + that).
                  The 2^-110 term covers __fdividef's zero result for denominators past 2^126 (|x| > 86), where the
                  exact value is below |x| 2^-124.
  epilogue        alpha, the two residual adds, gamma (or the one product by fl(alpha gamma)): four fp32 operations,
                  E = |alpha gamma| Ey (1 + 8u) + 4.04 u |gamma| (|alpha y| + |res1| + |res2|).
  fp16 stores     the interval map _rnd: a kernel value within E of v rounds to within max(h(v + E) - h(v), h(v) -
                  h(v - E)) of h(v) (h = fp16 rounding, monotone): zero where [v - E, v + E] holds no rounding boundary.
  out2            the same through lrelu (monotone, 1-Lipschitz), its fp32 product adding u |s v|.
Every written value must also be finite.  The bound is checked by the CPU negative controls: an fp32 emulation of the
kernel passes it, and it rejects references with one tap shifted by a row, the dilation off by one, the bias shifted by
one column, the GLU halves swapped, the last (partial) k-block dropped, the mask off by one row and out_row0 off by one.

Dispatch.  _predict restates sb_gemm's selection (tile width 32 / 64 / 128 / 256 from the device's SM count, TMA store or
direct store, the narrow-channel K-collapse, m_fast).  The case list covers every reachable (tile width, store path)
pair, both collapse outcomes and both m_fast outcomes (checked on the CPU at 132 and 114 SMs, the H100 SXM and PCIe), and
on the GPU torch.profiler records which gemm_tc_kernel<BN> each case launched.  The TMA store also needs a row of
n_out outputs to end on a 16-byte boundary: the bulk store writes a row's last 16-byte unit whole, so otherwise it
overwrites padding columns past n_out (the sentinel check of the tile-statistics case with out_ld = n + 2 shows it).

The tile-statistics and nearest-centroid bounds are derived where they are used."""
import contextlib
import ctypes
import json
import math
import os
import re
import tempfile
from dataclasses import dataclass, replace

import pytest
import torch

gpu = pytest.mark.gpu
dev = "cuda"
SB_OK, SB_EINVAL, SB_ENOSUP = 0, -1, -3  # include/seamless_b200.h
ACT_NONE, ACT_RELU, ACT_SILU, ACT_LRELU, ACT_TANH, ACT_GELU = range(6)
U32 = 2.0 ** -24          # fp32 unit roundoff
U_TC = 2.0 ** -23         # tensor-core fp32 accumulation (alignment / truncation): twice the round-to-nearest unit
SENT = -777.0             # exact in fp16 and fp32; no case computes it
BM, BK = 128, 64          # gemm_tcgen05.cu: tile rows, k-block depth
LEAD, TAIL = 8, 8         # NaN rows before and after A's addressable rows
OUT_TAIL = 5              # sentinel rows after the output window
SMS_CHECKED = (132, 114)  # H100 SXM, H100 PCIe


def _lib():
    from seamless_communication_b200 import _lib as L
    return L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gamma(n, unit):
    return n * unit / (1 - n * unit)


def _h(z):
    return z.half().double()


def _lrelu(z, s):
    return torch.where(z > 0, z, z * s)


def _rnd(v, E):
    """Kernel value fp16(v') with |v' - v| <= E, against the reference fp16(v): (reference, bound on the difference)."""
    r = _h(v)
    return r, torch.maximum(_h(v + E) - r, r - _h(v - E))


def _rnd_lrelu(v, E, s):
    """The same through lrelu (1-Lipschitz, monotone); the kernel's fp32 product z * s adds u |z s|."""
    r = _h(_lrelu(v, s))
    m = U32 * s * (v.abs() + E)
    return r, torch.maximum(_h(_lrelu(v + E, s) + m) - r, r - _h(_lrelu(v - E, s) - m))


# ================================================================================================ cases
@dataclass(frozen=True)
class Case:
    name: str
    m: int
    n: int
    c_in: int
    taps: int = 1
    dil: int = 1
    a_row0: int = 0
    a_rows: int = 0          # 0: a_row0 + m + (taps - 1) dil, every window inside A
    a_ld: int = 0            # 0: c_in
    act: int = ACT_NONE
    slope: float = 0.0
    glu: bool = False
    alpha: float = 1.0
    gamma: float = 1.0
    res: str = ""            # "1", "2" or "12"
    res_pad: int = 0         # res_ld = n_out + res_pad
    out_f32: bool = False
    out_pad: int = 0         # out_ld = n_out + out_pad
    out2: bool = False
    out2_pad: int = 0
    out2_slope: float = 0.125
    out_row0: int = 0
    seq: tuple = ()          # () no mask; (Tp, halo, T) with seq_lens NULL; (Tp, halo, None, lens) per sequence
    exact: bool = True
    bn256: bool = True       # SB_GEMM_BN256
    stats: bool = False      # tile_stats on the general kernel (SB_PROJ_T=0)

    @property
    def n_out(self):
        return self.n // 2 if self.glu else self.n

    @property
    def rows_a(self):
        return self.a_rows or self.a_row0 + self.m + (self.taps - 1) * self.dil

    @property
    def lda(self):
        return self.a_ld or self.c_in

    @property
    def out_rows(self):
        return self.out_row0 + self.m + OUT_TAIL

    def __str__(self):
        return self.name


M_BIG = 2 * 132 * BM + 77  # above two 128-row tiles per SM on both H100 variants
EXACT = [
    Case("m1_n8_direct", 1, 8, 8, out_pad=8),
    Case("m127_n20_f32_tma", 127, 20, 16, out_f32=True, out_pad=4, alpha=2.0, act=ACT_RELU),
    Case("m128_n40_collapse_out2_res1", 128, 40, 56, taps=3, a_row0=1, out2=True, res="1", res_pad=8, alpha=0.5),
    Case("m129_n72_taps7_clipped_res2", 129, 72, 72, taps=7, a_row0=-3, a_rows=129, res="2", res_pad=3, gamma=2.0),
    Case("m160_n136_dil5_seqlen", 160, 136, 136, taps=11, dil=5, a_row0=-25, a_rows=170, out_row0=3, seq=(80, 2, 70),
         act=ACT_LRELU, slope=0.125),
    Case("m256_n200_k1000_f32", 256, 200, 1000, out_f32=True, act=ACT_RELU, alpha=2.0, gamma=0.5),
    Case("m257_n264_dil3_res12_lens", 257, 264, 72, taps=3, dil=3, a_row0=-3, a_rows=257, res="12", res_pad=8,
         out_row0=5, seq=(80, 3, None, (74, 0, 1, 37)), act=ACT_LRELU, slope=0.125, alpha=0.5, gamma=2.0),
    Case("m257_n40_taps128_ald88", 257, 40, 80, taps=128, a_ld=88, a_row0=-64, a_rows=300, gamma=0.5),
    Case("m2000_n1032_bn128_tma", 2000, 1032, 64, act=ACT_RELU, out_row0=7),
    Case("m2000_n1032_bn128_direct", 2000, 1032, 64, out_pad=4, res="1", res_pad=4, alpha=0.5, out2=True, out2_pad=8),
    Case("m10000_n1024_bn256_tma", 10000, 1024, 64, taps=3, a_row0=-1, a_rows=10000, act=ACT_LRELU, slope=0.125,
         seq=(1000, 1, None, (998, 0, 1, 500, 998, 998, 0, 37, 998, 2))),
    Case("m10000_n1024_bn256_direct", 10000, 1024, 64, out_pad=4, res="1", alpha=2.0, gamma=0.5),
    Case("m10000_n1024_bn256_off", 10000, 1024, 64, taps=3, a_row0=-1, a_rows=10000, bn256=False),
    Case("mbig_n8_collapse_out2", M_BIG, 8, 8, taps=2, out2=True, out_row0=1),
    Case("m300_n136_bn64_direct", 300, 136, 64, out_pad=2, act=ACT_RELU),
    Case("m160_n64_bn32_f32_tma", 160, 64, 64, out_f32=True),
    # narrow channels (c_in < 64, a_ld == c_in, dilation 1): windows inside A take the K-collapse; windows that start
    # before row 0 or run past a_rows must read zeros for their outside taps only
    Case("narrow_c16_taps7_inside", 700, 16, 16, taps=7, a_row0=0),
    Case("narrow_c16_taps7_row0_neg", 700, 16, 16, taps=7, a_row0=-3, a_rows=700),
    Case("narrow_c32_taps11_tail_clipped", 300, 32, 32, taps=11, a_row0=2, a_rows=305),
    Case("narrow_c8_taps11_both_clipped", 260, 8, 8, taps=11, a_row0=-5, a_rows=260, out_f32=True),
]
BOUNDED = [
    Case("silu_res1_out2_lens", 300, 136, 136, taps=3, a_row0=-1, a_rows=300, act=ACT_SILU, res="1", alpha=0.5,
         gamma=1 / 3, out2=True, out2_slope=0.01, seq=(100, 1, None, (98, 37, 0)), exact=False),
    Case("glu_bn64_direct", 300, 136, 72, glu=True, exact=False),
    Case("glu_f32_bn128_direct", 2000, 2064, 64, glu=True, out_f32=True, exact=False),
    Case("gelu_bn256", 10000, 1024, 320, act=ACT_GELU, alpha=0.5, exact=False),
    Case("silu_bn256", 10000, 1280, 320, act=ACT_SILU, exact=False),
    Case("glu_bn256", 10000, 1024, 320, glu=True, res="1", alpha=0.5, exact=False),
    Case("tanh_f32_mfast", 160, 1032, 1024, act=ACT_TANH, out_f32=True, exact=False),
    Case("lrelu_res12_out2", 513, 72, 160, act=ACT_LRELU, slope=0.1, res="12", res_pad=8, out2=True, out2_slope=0.1,
         alpha=0.5, gamma=1 / 3, exact=False),
    Case("glu_bn32", 128, 40, 64, glu=True, out_row0=2, exact=False),
    Case("silu_k4096_bn128", 2000, 1032, 4096, act=ACT_SILU, exact=False),
]
STATS = [Case(f"stats_ld{20102 + p}", 300, 20102, 128, out_f32=True, out_pad=p, seq=(100, 0, None, (100, 37, 0)),
              exact=False, stats=True) for p in (0, 2)]
# the parent's K-collapse zero-filled whole windows at the buffer edges
COLLAPSE_EDGE = [c for c in EXACT if c.name.startswith("narrow_") and c.name != "narrow_c16_taps7_inside"]


def _predict(c, sms):
    """sb_gemm's kernel selection: (tile width, TMA store, K-collapse, m_fast)."""
    collapse = (c.taps > 1 and c.dil == 1 and c.c_in < BK and c.lda == c.c_in and c.a_row0 >= 0
                and c.a_row0 + c.m + c.taps - 1 <= c.rows_a)
    mt = -(-c.m // BM)

    def tiles(bn):
        return mt * -(-c.n // bn)

    if c.stats:
        bn = 128
    elif c.bn256 and c.n % 256 == 0 and not c.out_f32 and not c.out2 and tiles(256) >= 2 * sms:
        bn = 256
    elif c.n >= 128 and tiles(128) >= sms:
        bn = 128
    elif c.n >= 64 and tiles(64) >= sms:
        bn = 64
    elif c.n > 64:
        bn = 64
    else:
        bn = 32
    esize = 4 if c.out_f32 else 2
    nto = bn // 2 if c.glu else bn
    tma = (nto * esize >= 128 and ((c.n_out + c.out_pad) * esize) % 16 == 0 and (c.n_out * esize) % 16 == 0
           and not (c.glu and c.out_f32))
    if c.out2:
        tma = tma and ((c.n_out + c.out2_pad) * 2) % 16 == 0 and (c.n_out * 2) % 16 == 0 and nto >= 64
    return bn, tma, collapse, c.m <= 2 * BM and mt > 1


# ================================================================================================ inputs
def _seq_valid(c, q):
    """Sequence-mask validity of output rows q (int64 tensor)."""
    if not c.seq:
        return torch.ones_like(q, dtype=torch.bool)
    Tp, halo = c.seq[0], c.seq[1]
    b = q // Tp
    pos = q - b * Tp - halo
    if c.seq[2] is not None:
        ln = torch.full_like(q, c.seq[2])
    else:
        ln = torch.tensor(c.seq[3], dtype=torch.int64, device=q.device)[b.clamp(0, len(c.seq[3]) - 1)]
    return (pos >= 0) & (pos < ln)


def _make(c, device, seed=0):
    """Inputs and sentinel-filled outputs of one case; NaN wherever the call must not read."""
    g = torch.Generator(device=device).manual_seed(seed + 7919 * c.m + 31 * c.n + c.c_in)
    K = c.taps * c.c_in
    nan = float("nan")

    def grid(shape, lo, hi, den):
        return (torch.randint(lo, hi + 1, shape, generator=g, device=device).double() / den)

    def normal(shape, s=1.0):
        return torch.randn(shape, generator=g, device=device, dtype=torch.float64) * s

    A = torch.full((LEAD + c.rows_a + TAIL, c.lda), nan, dtype=torch.float16, device=device)
    W = torch.full((c.n + 8, K), nan, dtype=torch.float16, device=device)
    bias = torch.full((c.n + 8,), nan, dtype=torch.float32, device=device)
    if c.exact:
        A[LEAD:LEAD + c.rows_a, :c.c_in] = grid((c.rows_a, c.c_in), -4, 4, 4).half()
        W[:c.n] = grid((c.n, K), -4, 4, 8).half()
        bias[:c.n] = grid((c.n,), -64, 64, 32).float()
    else:
        A[LEAD:LEAD + c.rows_a, :c.c_in] = normal((c.rows_a, c.c_in)).half()
        W[:c.n] = normal((c.n, K), 40 / math.sqrt(K)).half()  # pre-activation std ~40
        bias[:c.n] = normal((c.n,)).float()
    t = dict(A=A, W=W, bias=bias)
    q = torch.arange(c.out_rows, device=device)
    live = (q >= c.out_row0) & (q < c.out_row0 + c.m) & _seq_valid(c, q)
    for r in c.res:
        ld = c.n_out + c.res_pad
        R = torch.full((c.out_rows, ld), nan, dtype=torch.float16, device=device)
        vals = grid((c.out_rows, c.n_out), -64, 64, 32) if c.exact else normal((c.out_rows, c.n_out))
        R[:, :c.n_out] = torch.where(live[:, None], vals, torch.full_like(vals, nan)).half()
        t["res" + r] = R
    t["out"] = torch.full((c.out_rows, c.n_out + c.out_pad), SENT, dtype=torch.float32 if c.out_f32 else torch.float16,
                          device=device)
    if c.out2:
        t["out2"] = torch.full((c.out_rows, c.n_out + c.out2_pad), SENT, dtype=torch.float16, device=device)
    if c.seq and c.seq[2] is None:
        t["lens"] = torch.tensor(c.seq[3], dtype=torch.int32, device=device)
        assert len(c.seq[3]) == (c.out_row0 + c.m - 1) // c.seq[0] + 1
    if c.stats:
        t["stats"] = torch.full((-(-c.n // 128), c.m, 2), nan, dtype=torch.float32, device=device)
    return t


def _desc(c, t, **override):
    from seamless_communication_b200._lib import GemmDesc
    d = GemmDesc()
    A = t["A"]
    d.a, d.a_rows, d.a_ld = A.data_ptr() + LEAD * A.stride(0) * 2, c.rows_a, A.stride(0)
    d.c_in, d.taps, d.dil, d.a_row0 = c.c_in, c.taps, c.dil, c.a_row0
    d.w, d.n, d.m = t["W"].data_ptr(), c.n, c.m
    d.bias, d.act, d.act_slope, d.glu = t["bias"].data_ptr(), c.act, c.slope, int(c.glu)
    d.alpha, d.gamma = c.alpha, c.gamma
    if "res1" in t:
        d.res1, d.res1_ld = t["res1"].data_ptr(), t["res1"].stride(0)
    if "res2" in t:
        d.res2, d.res2_ld = t["res2"].data_ptr(), t["res2"].stride(0)
    d.out, d.out_ld, d.out_f32 = t["out"].data_ptr(), t["out"].stride(0), int(c.out_f32)
    if "out2" in t:
        d.out2, d.out2_ld, d.out2_slope = t["out2"].data_ptr(), t["out2"].stride(0), c.out2_slope
    d.out_row0 = c.out_row0
    if c.seq:
        d.seq_rows, d.seq_halo = c.seq[0], c.seq[1]
        if c.seq[2] is not None:
            d.seq_len = c.seq[2]
        else:
            d.seq_lens = t["lens"].data_ptr()
    if "stats" in t:
        d.tile_stats = t["stats"].data_ptr()
    for k, v in override.items():
        setattr(d, k, v)
    return d


@contextlib.contextmanager
def _env(c):
    """SB_GEMM_BN256 and SB_PROJ_T are read per call."""
    keep = {k: os.environ.get(k) for k in ("SB_GEMM_BN256", "SB_PROJ_T")}
    os.environ["SB_GEMM_BN256"] = "1" if c.bn256 else "0"
    os.environ["SB_PROJ_T"] = "0"
    try:
        yield
    finally:
        for k, v in keep.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _call(c, t, ref=False):
    lib = _lib()
    with _env(c):
        rc = (lib.sb_gemm_ref if ref else lib.sb_gemm)(ctypes.byref(_desc(c, t)), _stream())
    assert rc == SB_OK, lib.sb_last_error()


# ================================================================================================ reference
def _act64(x, c):
    if c.act == ACT_RELU:
        return x.clamp_min(0)
    if c.act == ACT_LRELU:
        return _lrelu(x, c.slope)
    if c.act == ACT_SILU:
        return x * torch.sigmoid(x)
    if c.act == ACT_TANH:
        return torch.tanh(x)
    if c.act == ACT_GELU:
        return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    return x


def _act_bound(x, E0, c):
    """Bound on |kernel activation - f(x)| given |kernel pre-activation - x| <= E0 (module docstring)."""
    y = _act64(x, c)
    tiny = 2.0 ** -110 * (x.abs() + E0)
    if c.act == ACT_SILU:
        r = (4 + 1.173 * (x.abs() + E0)) * 2.0 ** -23 + U32
        return 1.1 * E0 + r * (y.abs() + 1.1 * E0) + tiny
    if c.act == ACT_GELU:
        xa = x.abs() + E0
        return 1.13 * E0 + 0.5 * xa * (2.0 ** -22 + 0.8 * U32 * xa + 2 * U32) + U32 * (y.abs() + 1.13 * E0) + tiny
    if c.act == ACT_TANH:
        return E0 + 2.0 ** -22 * (y.abs() + E0)
    if c.act == ACT_LRELU:
        return E0 + U32 * c.slope * (x.abs() + E0)
    return E0


def _reference(c, t, defect=None):
    """float64 contract -> (V, E): (out_rows, n_out) reference outputs and bounds (E = 0 on masked rows and in the exact
    family).  defect: one of the negative controls' wrong references."""
    A = t["A"][LEAD:LEAD + c.rows_a, :c.c_in].double()
    W = t["W"][:c.n].double()
    b = t["bias"][:c.n].double()
    if defect == "bias":
        b = torch.roll(b, -1)
    dil = c.dil + (1 if defect == "dil" else 0)
    x = torch.zeros((c.m, c.n), dtype=torch.float64, device=A.device)
    S = torch.zeros_like(x)
    rows = torch.arange(c.m, device=A.device) + c.a_row0
    for tap in range(c.taps):
        r = rows + tap * dil + (1 if defect == "tap" and tap == 0 else 0)
        ok = (r >= 0) & (r < c.rows_a)
        Ar = A[r.clamp(0, c.rows_a - 1)] * ok[:, None]
        Wt = W[:, tap * c.c_in:(tap + 1) * c.c_in]
        if defect == "kblock" and tap == c.taps - 1:
            Wt = Wt.clone()
            Wt[:, (c.c_in - 1) // BK * BK:] = 0
        x += Ar @ Wt.t()
        if not c.exact:
            S += Ar.abs() @ Wt.abs().t()
    x += b
    E0 = _gamma(c.taps * c.c_in + 2, U_TC) * (S + b.abs())
    if c.glu:
        a, g = (x[:, 1::2], x[:, 0::2]) if defect == "glu" else (x[:, 0::2], x[:, 1::2])
        Ea, Eg = E0[:, 0::2], E0[:, 1::2]
        y = a * torch.sigmoid(g)
        r = (4 + 1.173 * (g.abs() + Eg)) * 2.0 ** -23 + U32
        Ey0 = Ea + a.abs() * Eg / 4 + Ea * Eg / 4
        Ey = Ey0 + r * (y.abs() + Ey0) + 2.0 ** -110 * (a.abs() + Ea)
    else:
        y, Ey = _act64(x, c), _act_bound(x, E0, c)
    rs = [t["res" + k][:, :c.n_out].double() for k in c.res]
    row0 = c.out_row0 + (1 if defect == "row0" else 0)
    q = torch.arange(c.m, device=A.device) + row0
    R = [r[q] for r in rs]
    if R:
        V = (c.alpha * y + sum(R)) * c.gamma
    else:
        V = y * (c.alpha * c.gamma)
    E = abs(c.alpha * c.gamma) * Ey * (1 + 8 * U32) + 4.04 * U32 * abs(c.gamma) * (
        (c.alpha * y).abs() + sum((r.abs() for r in R), torch.zeros_like(y)))
    valid = _seq_valid(c, q)
    if defect == "mask":
        valid = _seq_valid(c, q) | _seq_valid(c, q - 1)  # one more row per sequence
    V = torch.where(valid[:, None], V, torch.zeros_like(V))
    E = torch.where(valid[:, None], E, torch.zeros_like(E))
    Vf = torch.zeros((c.out_rows, c.n_out), dtype=torch.float64, device=A.device)
    Ef = torch.zeros_like(Vf)
    Vf[row0:row0 + c.m], Ef[row0:row0 + c.m] = V, E
    return Vf, Ef


def _violations(c, got, V, E, slope=None):
    """Elements of one output (out, or out2 with its lrelu slope) outside the contract: a changed sentinel, a non-finite
    value, or a value outside the bound (exact family: any difference)."""
    ld = got.shape[1]
    win = torch.zeros(got.shape, dtype=torch.bool, device=got.device)
    win[c.out_row0:c.out_row0 + c.m, :c.n_out] = True
    bits = got.view(torch.int32 if got.dtype == torch.float32 else torch.int16)
    sent = torch.tensor(SENT, dtype=got.dtype).view(bits.dtype).item()
    bad = int((bits[~win] != sent).sum())
    g = got[c.out_row0:c.out_row0 + c.m, :c.n_out].double()
    v, e = V[c.out_row0:c.out_row0 + c.m], E[c.out_row0:c.out_row0 + c.m]
    bad += int((~torch.isfinite(g)).sum())
    if slope is not None:
        want, B = _rnd_lrelu(v, e, slope)
    elif got.dtype == torch.float16:
        want, B = _rnd(v, e)
    else:
        want, B = v, e
    if c.exact:
        B = torch.zeros_like(B)
    bad += int((~((g - want).abs() <= B)).sum())  # a NaN reference (a residual canary read) counts
    assert ld >= c.n_out
    return bad


def _check(c, t, V, E, what):
    bad = _violations(c, t["out"], V, E)
    assert bad == 0, f"{what}: {bad} wrong elements of out"
    if c.out2:
        bad = _violations(c, t["out2"], V, E, c.out2_slope)
        assert bad == 0, f"{what}: {bad} wrong elements of out2"


# ================================================================================================ CPU tests
def test_dispatch_table_covers_every_cell():
    """The cases reach every (tile width, store path) pair sb_gemm can select, the K-collapse and the per-tap path on
    narrow channels, and m_fast on and off, at the SM counts of both H100 variants."""
    for sms in SMS_CHECKED:
        seen = {_predict(c, sms) for c in EXACT + BOUNDED + STATS}
        cells = {(bn, tma) for bn, tma, _, _ in seen}
        assert cells == {(bn, tma) for bn in (32, 64, 128, 256) for tma in (False, True)}, (sms, cells)
        assert {s[2] for s in seen} == {False, True} and {s[3] for s in seen} == {False, True}, sms
        for c in COLLAPSE_EDGE:
            assert not _predict(c, sms)[2], c  # the windows at the edges keep the per-tap path
    narrow = [c for c in EXACT if c.name.startswith("narrow_")]
    assert {_predict(c, 132)[2] for c in narrow} == {False, True}


def _emulate(c, t):
    """The kernel's arithmetic in fp32 on the CPU: fp32 accumulation, the fp32 activation, the epilogue's fp32
    operations in the kernel's order, fp16 stores; outputs in the sentinel-filled buffers of t."""
    A = t["A"][LEAD:LEAD + c.rows_a, :c.c_in].float()
    W = t["W"][:c.n].float()
    x = torch.zeros((c.m, c.n), dtype=torch.float32)
    rows = torch.arange(c.m) + c.a_row0
    for tap in range(c.taps):
        r = rows + tap * c.dil
        ok = (r >= 0) & (r < c.rows_a)
        x += (A[r.clamp(0, c.rows_a - 1)] * ok[:, None]) @ W[:, tap * c.c_in:(tap + 1) * c.c_in].t()
    x = x + t["bias"][:c.n]
    if c.glu:
        y = x[:, 0::2] / (1 + torch.exp(-x[:, 1::2]))
    elif c.act == ACT_SILU:
        y = x / (1 + torch.exp(-x))
    elif c.act == ACT_GELU:
        y = 0.5 * x * (1 + torch.erf(x * 0.70710678118654752))
    elif c.act == ACT_TANH:
        y = torch.tanh(x)
    elif c.act == ACT_LRELU:
        y = torch.where(x > 0, x, x * c.slope)
    elif c.act == ACT_RELU:
        y = x.clamp_min(0)
    else:
        y = x
    q = torch.arange(c.m) + c.out_row0
    if c.res:
        y = y * c.alpha
        for k in c.res:
            y = y + t["res" + k][q, :c.n_out].float()
        y = y * c.gamma
    else:
        y = y * torch.tensor(c.alpha, dtype=torch.float32) * torch.tensor(c.gamma, dtype=torch.float32)
    y = torch.where(_seq_valid(c, q)[:, None], y, torch.zeros_like(y))
    t["out"][c.out_row0:c.out_row0 + c.m, :c.n_out] = y.to(t["out"].dtype)
    if c.out2:
        t["out2"][c.out_row0:c.out_row0 + c.m, :c.n_out] = torch.where(y > 0, y, y * c.out2_slope).half()


CONTROL = Case("control", 150, 72, 136, taps=3, dil=2, a_row0=-2, a_rows=151, glu=True, res="12", res_pad=8, alpha=0.5,
               gamma=1 / 3, out2=True, out2_slope=0.01, out_row0=3, seq=(40, 2, None, (36, 20, 0, 7)), exact=False)


@pytest.mark.parametrize("defect", [None, "tap", "dil", "bias", "glu", "kblock", "mask", "row0"])
def test_bound_accepts_emulation_and_rejects_wrong_references(defect):
    """An fp32 emulation of the kernel passes the bounded-family check against the float64 contract; the same check
    rejects it against each wrong reference (c_in = 136 leaves a partial last k-block of 8 channels)."""
    for c in (CONTROL, replace(CONTROL, glu=False, act=ACT_SILU, name="control_silu"),
              replace(CONTROL, glu=False, act=ACT_GELU, out_f32=True, out2=False, name="control_gelu")):
        if defect == "glu" and not c.glu:
            continue
        t = _make(c, "cpu")
        _emulate(c, t)
        V, E = _reference(c, t, defect)
        bad = _violations(c, t["out"], V, E)
        if defect is None:
            assert bad == 0, c
            if c.out2:
                assert _violations(c, t["out2"], V, E, c.out2_slope) == 0, c
        else:
            assert bad > 0, (c, defect)


# ================================================================================================ GPU tests
@gpu
@pytest.mark.parametrize("c", EXACT, ids=str)
def test_gemm_exact_family(c):
    """Exact inputs: sb_gemm and the CUDA-core sb_gemm_ref equal the float64 contract bit for bit, canaries unread and
    sentinels intact (one launch each)."""
    t = _make(c, dev)
    V, E = _reference(c, t)
    n0 = _lib().sb_launch_count()
    _call(c, t)
    assert _lib().sb_launch_count() == n0 + 1
    torch.cuda.synchronize()
    _check(c, t, V, E, "sb_gemm")
    t = _make(c, dev)
    _call(c, t, ref=True)
    torch.cuda.synchronize()
    _check(c, t, V, E, "sb_gemm_ref")


@gpu
@pytest.mark.parametrize("c", BOUNDED, ids=str)
def test_gemm_bounded_family(c):
    """Full-mantissa inputs at production scales: every output within the per-element bound of the module docstring."""
    t = _make(c, dev)
    V, E = _reference(c, t)
    _call(c, t)
    torch.cuda.synchronize()
    _check(c, t, V, E, "sb_gemm")


def _launched_tiles(cases):
    """The gemm_tc_kernel<BN> instantiation each case launches, in order, from a torch.profiler trace."""
    from torch.profiler import ProfilerActivity, profile
    inputs = [_make(c, dev) for c in cases]
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for c, t in zip(cases, inputs):
                _call(c, t)
                torch.cuda.synchronize()
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    ks = sorted((e["ts"], e["name"]) for e in ev if e.get("cat") == "kernel" and "gemm_tc_kernel" in e.get("name", ""))
    return [int(re.search(r"gemm_tc_kernel<(\d+)>", n).group(1)) for _, n in ks]


@gpu
def test_dispatch_matches_profiled_kernels():
    """Every case launches the tile width _predict gives at this device's SM count (SB_GEMM_BN256=0 moves a 256-eligible
    case to 128-wide tiles; tile statistics on the general kernel are per 128 columns)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cases = EXACT + BOUNDED + STATS
    got = _launched_tiles(cases)
    want = [_predict(c, sms)[0] for c in cases]
    assert got == want, (sms, [(c.name, g, w) for c, g, w in zip(cases, got, want) if g != w])


@gpu
@pytest.mark.parametrize("c", STATS, ids=str)
def test_tile_stats_general_kernel(c):
    """tile_stats on the general kernel (SB_PROJ_T=0) at 300 rows over 158 column tiles (the last one 6 wide), with
    masked rows: the max is the max of the stored fp32 logits bit for bit; the sum of exp(x - max) is within
      sum_j e^{x_j} (4 ((2 + 1.173 |x_j|) 2^-23 + u |x_j|)) + gamma_40(u) S + 128 * 2^-126.
    Each term passes through at most four __expf (its own and up to three rescales of the running sum by
    __expf(old max - new max), whose arguments are no larger in magnitude than x_j), each after an fp32 subtraction; the
    32-term chunk sums and the rescale products add gamma_40(u) of the total; results flushed below 2^-126 add the last
    term."""
    t = _make(c, dev)
    V, E = _reference(c, t)
    _call(c, t)
    torch.cuda.synchronize()
    _check(c, t, V, E, "sb_gemm")
    L = t["out"][c.out_row0:c.out_row0 + c.m, :c.n].double()
    st = t["stats"].double()
    nt = st.shape[0]
    pad = nt * 128 - c.n
    Lp = torch.cat([L, torch.full((c.m, pad), -math.inf, dtype=torch.float64, device=dev)], 1).view(c.m, nt, 128)
    mx = Lp.max(-1).values.t()
    assert torch.equal(st[..., 0], mx)
    x = Lp - mx.t()[..., None]
    ex = torch.exp(x)
    S = ex.sum(-1).t()
    xa = torch.where(torch.isfinite(x), x.abs(), torch.zeros_like(x))
    err = (ex * 4 * ((2 + 1.173 * xa) * 2.0 ** -23 + U32 * xa)).sum(-1).t() + _gamma(40, U32) * S + 128 * 2.0 ** -126
    assert ((st[..., 1] - S).abs() <= err).all(), ((st[..., 1] - S).abs() / err).max().item()
    rows_masked = ~_seq_valid(c, torch.arange(c.m, device=dev))
    assert (st[:, rows_masked, 0] == 0).all()


@gpu
@pytest.mark.parametrize("K", [1, 5, 127, 129])
def test_nearest_centroid_exact(K):
    """sb_nearest_centroid in the exact family (dim 72, x and centroids on the 1/4 grid in [-1, 1], |c|^2 / 2 exact in
    fp32): the unit of every valid row is the lowest index of its minimum distance, computed exactly; duplicated
    centroids inside a 128-column tile and across tiles make ties; masked rows give -1.  Columns 72..79 of x are NaN."""
    lib = _lib()
    g = torch.Generator(device="cpu").manual_seed(K)
    dim, ld, Tp, lens = 72, 80, 100, (100, 37, 0)
    rows = Tp * len(lens)
    cen = torch.randint(-4, 5, (K, dim), generator=g).double() / 4
    if K >= 5:
        cen[3] = cen[1]
    if K == 129:
        cen[128] = cen[2]
        cen[100] = cen[2]
    x = torch.randint(-4, 5, (rows, dim), generator=g).double() / 4
    pick = torch.randint(0, K, (rows // 2,), generator=g)
    x[: rows // 2] = cen[pick]  # distance 0 to a (possibly duplicated) centroid
    xb = torch.full((rows, ld), float("nan"), dtype=torch.float16)
    xb[:, :dim] = x.half()
    nh = (-0.5 * (cen * cen).sum(1)).float()
    d = (cen * cen).sum(1)[None] - 2 * x @ cen.t()  # |x - c|^2 - |x|^2, exact
    want = d.argmin(1).int()  # first minimum
    dmin = d.min(1, keepdim=True).values
    first = torch.stack([torch.nonzero(d[r] == dmin[r])[0, 0] for r in range(rows)]).int()
    assert torch.equal(want, first)
    pos = torch.arange(rows) % Tp
    valid = pos < torch.tensor(lens)[torch.arange(rows) // Tp]
    want = torch.where(valid, want, torch.full_like(want, -1))
    xd, cd, nd = xb.to(dev), cen.half().to(dev), nh.to(dev)
    ln = torch.tensor(lens, dtype=torch.int32, device=dev)
    best = torch.empty((rows,), dtype=torch.int64, device=dev)
    units = torch.full((rows,), -7, dtype=torch.int32, device=dev)
    rc = lib.sb_nearest_centroid(xd.data_ptr(), ld, rows, dim, cd.data_ptr(), nd.data_ptr(), K, Tp, ln.data_ptr(),
                                 best.data_ptr(), units.data_ptr(), _stream())
    assert rc == SB_OK, lib.sb_last_error()
    assert torch.equal(units.cpu(), want)


@gpu
@pytest.mark.parametrize("what", ["out", "out2", "res1", "res2", "stats_f16", "rows"])
def test_refusals(what):
    """Calls outside the contract return SB_EINVAL before anything is launched, and write nothing: out / out2 / res1 /
    res2 8 bytes past a 16-byte boundary (row strides that are multiples of 8 elements, which the direct store's
    16-byte accesses would otherwise trust), tile_stats with an fp16 output, and m = 65536 * 128 rows, one more row tile
    than gridDim.y holds (real 134 MB A and out buffers, so even a launch could not write out of bounds)."""
    lib = _lib()
    if what == "rows":
        m = 65536 * BM
        c = Case("rows", m, 8, 8)
        t = dict(A=torch.zeros((LEAD + m + TAIL, 8), dtype=torch.float16, device=dev),
                 W=torch.zeros((16, 8), dtype=torch.float16, device=dev), bias=torch.zeros(16, device=dev),
                 out=torch.full((m + OUT_TAIL, 8), SENT, dtype=torch.float16, device=dev))
        d, text = _desc(c, t), "65535"
    else:
        c = Case(what, 128, 256 if what == "stats_f16" else 64, 64, res="12" if what.startswith("res") else "",
                 out2=what == "out2", out_pad=8, out2_pad=8, stats=what == "stats_f16", exact=False)
        t = _make(c, dev)
        if what == "stats_f16":
            d, text = _desc(c, t), "tile_stats needs out_f32"
        else:
            d, text = _desc(c, t, **{what: t[what].data_ptr() + 8}), "16B aligned"
    outs = [t[k].clone() for k in ("out", "out2") if k in t]
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    with _env(c):
        rc = lib.sb_gemm(ctypes.byref(d), _stream())
    torch.cuda.synchronize()
    assert rc == SB_EINVAL, (what, rc, lib.sb_last_error())
    assert text in lib.sb_last_error().decode()
    assert lib.sb_launch_count() == n0
    for o, k in zip(outs, ("out", "out2")):
        assert torch.equal(o.view(torch.int16) if o.dtype == torch.float16 else o.view(torch.int32),
                           t[k].view(torch.int16) if o.dtype == torch.float16 else t[k].view(torch.int32))
