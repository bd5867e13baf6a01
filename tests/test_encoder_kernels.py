"""The speech encoder's and the T2U's non-GEMM kernels, called through the C-ABI and checked against float64 torch
references built on the GPU from the kernels' own fp16 inputs.

sb_attention (csrc/attention.cu): plain, causal, Shaw and Shaw + causal self-attention, cross-attention with separate q
and kv buffers, the T2U's halo-3 layout.  The 64-row kernel (the default) runs in this process; the 128-row kernel
(SB_ATTENTION_V2=1, read once per process) runs the same case list in a child process.
sb_layernorm / sb_splitk_reduce_ln (csrc/layernorm.cu): every dim class, the warps-per-block switch, the residual and
its sum output, the asymmetric in / out layouts, the padding mask, split counts the engine can reach.
sb_dwconv_ln_silu (csrc/dwconv.cu): the 32-frame tile kernel (k = 31, C % 64 == 0), the fixed-31 kernel (C % 64 != 0
here, and SB_DWCONV_TILE=0 in a child process) and the generic-k kernel.

Inputs no kernel may read (halo rows, key / value rows past a sequence's length, table rows past the window) hold NaN,
and every output element outside the written region holds a sentinel that must survive bit for bit.  A sequence
computed alone must equal the same sequence computed in the batch bit for bit, and repeated calls are bit-identical.

The float64 references take the fp16 inputs as exact; what is left is the kernels' fp32 arithmetic and the final fp16
rounding (half an fp16 ulp: 2^-11 relative).  u = 2^-24 is the fp32 unit roundoff.  Each bound is derived where it is
used."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"
HD = 64
SB_OK, SB_ENOSUP = 0, -3  # include/seamless_b200.h
U32 = 2.0 ** -24          # fp32 unit roundoff
SENT = -777.0             # exact in fp16; no kernel ever computes it from these inputs
SENT_BITS = torch.tensor(SENT, dtype=torch.float16).view(torch.int16).item()


def _lib():
    from seamless_communication_b200 import _lib as L
    return L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(torch.int16)


def _child(func, env_var, value="1"):
    """Runs `test_encoder_kernels.<func>()` in a fresh process with env_var set: the kernel switches are read once."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; "
            f"import test_encoder_kernels as t; t.{func}(); print('ok')")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=900,
                       env={**os.environ, env_var: value})
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]


# ================================================================================================ sb_attention
def _attn_ref(q, k, v, causal_off, rel, relk):
    """float64 softmax((q.k^T + q.rel_k[clamp(j - i, -L, R) + L]) / 8) . v for one sequence.  q (sq, H, 64), k / v (n, H,
    64) float64 with n the key length; key j is admissible for query i iff j <= i + causal_off (causal_off None: all).
    Returns (out (sq, H, 64), empty (sq,) bool: rows without an admissible key, which the kernels write as 0)."""
    sq, H, _ = q.shape
    n = k.shape[0]
    i = torch.arange(sq, device=dev)[:, None]
    j = torch.arange(n, device=dev)[None, :]
    allowed = torch.ones(sq, n, dtype=torch.bool, device=dev) if causal_off is None else j <= i + causal_off
    empty = ~allowed.any(1)
    out = torch.zeros(sq, H, HD, dtype=torch.float64, device=dev)
    if n == 0:
        return out, empty
    idx = None if rel is None else ((j - i).clamp(-rel[0], rel[1]) + rel[0])
    chunk = max(1, (1 << 24) // (sq * n))  # heads per pass: (chunk, sq, n) float64 stays at or below 128 MB
    for h0 in range(0, H, chunk):
        hs = slice(h0, min(H, h0 + chunk))
        qh = q[:, hs].transpose(0, 1)                            # (h, sq, 64)
        s = qh @ k[:, hs].permute(1, 2, 0)                       # (h, sq, n)
        if rel is not None:
            qr = qh @ relk.t()                                   # (h, sq, L + R + 1)
            s += torch.gather(qr, 2, idx.expand(qh.shape[0], sq, n))
        s = (s / 8.0).masked_fill_(~allowed, -math.inf)
        p = torch.softmax(s, -1).nan_to_num_(0.0)                # rows with no admissible key: 0
        out[:, hs] = (p @ v[:, hs].transpose(0, 1)).transpose(0, 1)
    return out, empty


def _attn_case(sq, sk, H, lens, *, causal=False, rel=None, halo=0, kv_halo=None, tail=0, fused=True, scale=1.0, seed=0):
    """One sb_attention call checked against float64.  lens: per-sequence key lengths, or an int B for kv_lens = NULL.
    fused: q | k | v share one (rows, 3M) buffer (self-attention); otherwise q is (rows, M) and k | v one (rows, 2M)
    buffer with its own halo (cross-attention, as decode_full passes them) and `out` has 64 padding columns.  tail: extra
    rows per sequence past the halo that nobody writes (out_rows != sq + 2 halo)."""
    lib = _lib()
    B = lens if isinstance(lens, int) else len(lens)
    kvh = halo if kv_halo is None else kv_halo
    M = H * HD
    q_rows, kv_rows = sq + 2 * halo + tail, sk + 2 * kvh + tail
    g = torch.Generator(device=dev).manual_seed(seed * 7919 + sq * 131 + sk * 17 + H * 3 + halo + 5 * kvh)
    klen = [sk] * B if isinstance(lens, int) else [min(n, sk) for n in lens]
    if fused:
        assert sq == sk and kvh == halo
        buf = torch.randn(B, q_rows, 3 * M, device=dev, generator=g)
        buf[..., :M] *= scale
        buf = buf.half()
        qb, kb, vb = buf[..., :M], buf[..., M:2 * M], buf[..., 2 * M:]
        ob = torch.full((B, q_rows, M), SENT, dtype=torch.float16, device=dev)
    else:
        qb = (torch.randn(B, q_rows, M, device=dev, generator=g) * scale).half()
        kvb = torch.randn(B, kv_rows, 2 * M, device=dev, generator=g).half()
        kb, vb = kvb[..., :M], kvb[..., M:]
        ob = torch.full((B, q_rows, M + 64), SENT, dtype=torch.float16, device=dev)
    # poison: q halo rows, and k / v outside [kv_halo, kv_halo + len) of each sequence
    qb[:, :halo] = math.nan
    qb[:, halo + sq:] = math.nan
    for b in range(B):
        kb[b, :kvh] = kb[b, kvh + klen[b]:] = math.nan
        vb[b, :kvh] = vb[b, kvh + klen[b]:] = math.nan
    relk = None
    if rel is not None:
        nrel = rel[0] + rel[1] + 1
        relk = torch.full((nrel + 8, HD), math.nan, dtype=torch.float16, device=dev)  # rows past the window: NaN
        relk[:nrel] = (torch.randn(nrel, HD, device=dev, generator=g) * 0.5).half()
    lens_d = None if isinstance(lens, int) else torch.tensor(lens, dtype=torch.int32, device=dev)

    def call(b0, nb, out):
        rc = lib.sb_attention(qb[b0].data_ptr(), qb.stride(1), kb[b0].data_ptr(), kb.stride(1), vb[b0].data_ptr(),
                              vb.stride(1), out.data_ptr(), out.stride(1), nb, H, sq, sk, q_rows, halo, kv_rows, kvh,
                              None if lens_d is None else lens_d[b0:].data_ptr(), int(causal),
                              None if relk is None else relk.data_ptr(), rel[0] if rel else 0, rel[1] if rel else 0,
                              _stream())
        assert rc == SB_OK, lib.sb_last_error()

    call(0, B, ob)
    what = (f"sq={sq} sk={sk} H={H} lens={lens} causal={causal} rel={rel} halo={halo}/{kvh} tail={tail} "
            f"fused={fused} scale={scale}")
    # nothing outside rows [halo, halo + sq) x columns [0, M) of each sequence is written
    written = torch.zeros(ob.shape, dtype=torch.bool, device=dev)
    written[:, halo:halo + sq, :M] = True
    assert (_bits(ob)[~written] == SENT_BITS).all(), f"{what}: wrote outside the output rows"
    for b in range(B):
        n = klen[b]
        q64 = qb[b, halo:halo + sq].double().view(sq, H, HD)
        k64 = kb[b, kvh:kvh + n].double().view(n, H, HD)
        v64 = vb[b, kvh:kvh + n].double().view(n, H, HD)
        ref, empty = _attn_ref(q64, k64, v64, sk - sq if causal else None, rel, None if relk is None else relk[:nrel].double())
        got = ob[b, halo:halo + sq, :M].view(sq, H, HD)
        assert torch.isfinite(got).all(), f"{what} b={b}: non-finite output (a NaN row was read)"
        assert (got[empty] == 0).all(), f"{what} b={b}: a row without an admissible key is not 0"
        # Bound 2^-11 |ref| + 2^-11 max|v| + 1e-5 (test_v1_encoder's relpos test): fp16 output rounding; the softmax
        # weights exp(s - m) are rounded to fp16 before P.V (2^-11 relative each, against the fp32 row sum:
        # <= 2^-11 max|v|); scores are fp32 sums of 64 (+ 64 for the bias) products and __expf, inside 1e-5.
        vmax = v64.abs().max().item() if n else 0.0
        err = (got.double() - ref).abs()
        bound = 2.0 ** -11 * ref.abs() + 2.0 ** -11 * vmax + 1e-5
        worst = (err / bound).max().item()
        assert worst <= 1.0, f"{what} b={b}: error {err.max().item():.3e} is {worst:.2f}x the bound"
    # each sequence alone equals the same sequence in the batch, bit for bit (sentinel rows included)
    for b in range(B):
        one = torch.full_like(ob[:1], SENT)
        call(b, 1, one)
        assert torch.equal(_bits(one[0]), _bits(ob[b])), f"{what}: sequence {b} alone differs from the batch"
    again = torch.full_like(ob, SENT)
    call(0, B, again)
    assert torch.equal(_bits(again), _bits(ob)), f"{what}: repeated call differs"


SELF_S = (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 499, 500, 1000, 2048, 4096)
WINDOWS = ((0, 0), (79, 0), (0, 79), (3, 5), (2, 34), (66, 13))  # with (64, 8): nrel 1 .. 80; left / right 2 and 34
CROSS_SQ = (1, 5, 37, 102)
CROSS_SK = (1, 63, 64, 65, 190, 499, 752)
CAUSAL_DELTA = (-37, -1, 1, 37)
T2U_U = (1, 63, 64, 65, 300, 1000)


def _ragged(S):
    """Lengths 0, 1 and S in one batch, plus a length that ends inside a key block."""
    return [S, 0, 1, max(1, 2 * S // 3)]


def _self_cases(S, H):
    yield dict(sq=S, sk=S, H=H, lens=_ragged(S))
    yield dict(sq=S, sk=S, H=H, lens=_ragged(S), causal=True, scale=4.0)
    yield dict(sq=S, sk=S, H=H, lens=_ragged(S), rel=(64, 8))
    yield dict(sq=S, sk=S, H=H, lens=2, rel=(64, 8), causal=True, scale=4.0)


def _window_cases(window):
    for S in (65, 256, 700):
        yield dict(sq=S, sk=S, H=2, lens=_ragged(S), rel=window)
        yield dict(sq=S, sk=S, H=2, lens=_ragged(S), rel=window, causal=True, scale=4.0)


def _causal_offset_cases(delta):
    for sq in (1, 40, 130, 300):
        sk = sq + delta
        if sk < 1:
            continue
        yield dict(sq=sq, sk=sk, H=2, lens=[sk, 0, max(1, sk // 2)], causal=True, fused=False, kv_halo=2)
        yield dict(sq=sq, sk=sk, H=2, lens=2, causal=True, rel=(64, 8), fused=False, kv_halo=2, scale=4.0)


def _cross_cases(sk):
    for sq in CROSS_SQ:
        for lens in ([sk, 1, 0, max(1, sk // 2)], 3):  # per-sequence lengths, and kv_lens = NULL (monotonic decoder)
            for scale in (1.0, 4.0):
                yield dict(sq=sq, sk=sk, H=2, lens=lens, fused=False, halo=1, kv_halo=4, tail=3, scale=scale)


def _t2u_cases(U):
    yield dict(sq=U, sk=U, H=2, lens=_ragged(U), halo=3)
    yield dict(sq=U, sk=U, H=16, lens=_ragged(U), halo=3, scale=4.0)


def _all_attn_cases():
    for S in SELF_S:
        for H in (1, 2, 16):
            yield from _self_cases(S, H)
    for w in WINDOWS:
        yield from _window_cases(w)
    for d in CAUSAL_DELTA:
        yield from _causal_offset_cases(d)
    for sk in CROSS_SK:
        yield from _cross_cases(sk)
    for U in T2U_U:
        yield from _t2u_cases(U)


@pytest.mark.parametrize("H", [1, 2, 16])
@pytest.mark.parametrize("S", SELF_S)
def test_attention_self(S, H):
    """Plain, causal (q x 4: nearly one-hot softmax), Shaw (64, 8) as shipped, Shaw + causal with kv_lens = NULL."""
    for case in _self_cases(S, H):
        _attn_case(**case)


@pytest.mark.parametrize("window", WINDOWS)
def test_attention_shaw_windows(window):
    """Windows from a single row to the 80-row table: the clamp at both ends, and key blocks wholly left of, wholly
    right of and across every row's window (S >= 256: a 32- or 64-row group of queries sits wholly on one side)."""
    for case in _window_cases(window):
        _attn_case(**case)


@pytest.mark.parametrize("delta", CAUSAL_DELTA)
def test_attention_causal_bottom_right(delta):
    """Causal with sk != sq: key j is admissible for query i iff j <= i + sk - sq; for sk < sq the first sq - sk rows
    have no admissible key and are written as 0."""
    for case in _causal_offset_cases(delta):
        _attn_case(**case)


@pytest.mark.parametrize("sk", CROSS_SK)
def test_attention_cross(sk):
    """sq != sk from separate q (ld M) and k | v (ld 2M) buffers with different halos, out rows beyond the written
    region, kv_lens given and NULL."""
    for case in _cross_cases(sk):
        _attn_case(**case)


@pytest.mark.parametrize("U", T2U_U)
def test_attention_t2u_layout(U):
    """The T2U FFT decoder's layout: halo 3 on q, k / v and out, per-row lengths."""
    for case in _t2u_cases(U):
        _attn_case(**case)


def _attn_sweep():
    for case in _all_attn_cases():
        _attn_case(**case, seed=1)
    torch.cuda.synchronize()


def test_attention_128_row_kernel():
    """The same case list on attention2_kernel (SB_ATTENTION_V2=1), in a child process."""
    _child("_attn_sweep", "SB_ATTENTION_V2")


@pytest.mark.parametrize("what", ["rel_81", "rel_80_0", "rel_0_80", "q_ld", "k_ld", "v_ld"])
def test_attention_refusals(what):
    """A Shaw table of more than 80 rows, or q / k / v row strides that are not multiples of 8 elements, return
    SB_ENOSUP before anything is launched."""
    lib = _lib()
    H, S, M = 2, 70, 128
    buf = torch.zeros(S, 3 * M + 8, dtype=torch.float16, device=dev)
    out = torch.full((S, M), SENT, dtype=torch.float16, device=dev)
    relk = torch.zeros(96, HD, dtype=torch.float16, device=dev)
    left, right = {"rel_81": (46, 34), "rel_80_0": (80, 0), "rel_0_80": (0, 80)}.get(what, (64, 8))
    ld = {w: 3 * M + (4 if what == w else 0) for w in ("q_ld", "k_ld", "v_ld")}
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    rc = lib.sb_attention(buf.data_ptr(), ld["q_ld"], buf[:, M:].data_ptr(), ld["k_ld"], buf[:, 2 * M:].data_ptr(),
                          ld["v_ld"], out.data_ptr(), M, 1, H, S, S, S, 0, S, 0, None, 0, relk.data_ptr(), left, right,
                          _stream())
    torch.cuda.synchronize()
    assert rc == SB_ENOSUP, rc
    assert lib.sb_launch_count() == n0
    assert (_bits(out) == SENT_BITS).all()


# ================================================================================================ LayerNorm
def _ln_bound(ref, xhat, sd, xmax, w, b, dim):
    """|y - ref| for y = (v - mean) * rstd * w + b in fp32 from exact inputs v, with two-pass statistics whose sums run
    along at most n = dim / 32 + 21 sequential fp32 additions (a lane's share, at least 8 values, a 5-level shuffle
    tree, up to 8 cross-warp partials): |d mean| <= n u max|v| (first-order gamma bound); the centred sum of squares and rsqrt add
    (n + 8) u relative to var, i.e. (n / 2 + 4) u relative to x^; the subtraction and the two products and the add of
    the affine step 4 u.  Hence |d x^| <= u (n max|v| / sd + (n / 2 + 8) |x^|), and |y - ref| <= 2^-11 |ref| +
    |w| |d x^| + u (|w x^| + |b|)."""
    n = dim / 32 + 21
    dx = U32 * (n * xmax / sd + (n / 2 + 8) * xhat.abs())
    return 2.0 ** -11 * ref.abs() + w.abs() * dx + U32 * ((w * xhat).abs() + b.abs())


def _ln_ref(v, w, b):
    """float64 LayerNorm over the last dim (eps 1e-5): (ref, x^, sd, max|v|) per row."""
    mean = v.mean(-1, keepdim=True)
    sd = ((v - mean) ** 2).mean(-1, keepdim=True).add(1e-5).sqrt()
    xhat = (v - mean) / sd
    return xhat * w + b, xhat, sd, v.abs().amax(-1, keepdim=True)


def _ln_case(dim, B, T, *, in_halo=0, in_rows=None, out_halo=0, out_rows=None, res=False, lens=None, mask=False,
             offset=0.0, seed=0):
    lib = _lib()
    in_rows = T + 2 * in_halo if in_rows is None else in_rows
    out_rows = T + 2 * out_halo if out_rows is None else out_rows
    g = torch.Generator(device=dev).manual_seed(seed * 7919 + dim * 31 + B * 7 + T + in_halo + 3 * out_halo)
    x = (offset + torch.randn(B, in_rows, dim, device=dev, generator=g)).half()
    r = torch.randn(B, in_rows, dim, device=dev, generator=g).half() if res else None
    for t in (x, r):  # rows outside the sequences' data are never read
        if t is not None:
            t[:, :in_halo] = math.nan
            t[:, in_halo + T:] = math.nan
    w = torch.rand(dim, device=dev, generator=g) + 0.5
    bb = torch.randn(dim, device=dev, generator=g) * 0.2
    y = torch.full((B, out_rows, dim), SENT, dtype=torch.float16, device=dev)
    so = torch.full_like(y, SENT) if res else None
    lens_d = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    rc = lib.sb_layernorm(x.data_ptr(), None if r is None else r.data_ptr(), y.data_ptr(), None if so is None else so.data_ptr(),
                          w.data_ptr(), bb.data_ptr(), dim, B, T, in_rows, in_halo, out_rows, out_halo,
                          None if lens_d is None else lens_d.data_ptr(), int(mask), _stream())
    assert rc == SB_OK, lib.sb_last_error()
    assert lib.sb_launch_count() == n0 + 1
    what = f"dim={dim} B={B} T={T} in={in_rows}/{in_halo} out={out_rows}/{out_halo} res={res} lens={lens} mask={mask} offset={offset}"
    outside = torch.ones(B, out_rows, dim, dtype=torch.bool, device=dev)
    outside[:, out_halo:out_halo + T] = False
    assert (_bits(y)[outside] == SENT_BITS).all(), f"{what}: wrote outside the output rows"
    xd = x[:, in_halo:in_halo + T]
    if res:
        # sum_out is x + res summed in fp32 and rounded once, written in the OUT layout
        assert (_bits(so)[outside] == SENT_BITS).all(), f"{what}: sum_out written outside the output rows"
        assert torch.equal(_bits(so[:, out_halo:out_halo + T]), _bits((xd.float() + r[:, in_halo:in_halo + T].float()).half())), \
            f"{what}: sum_out"
    # the statistics see x + res in fp32 without rounding: the float64 sum is exact, the fp32 one is within u of it
    v = xd.double() + (r[:, in_halo:in_halo + T].double() if res else 0.0)
    ref, xhat, sd, vmax = _ln_ref(v, w.double(), bb.double())
    got = y[:, out_halo:out_halo + T]
    keep = torch.ones(B, T, dtype=torch.bool, device=dev)
    if mask and lens is not None:
        keep = torch.arange(T, device=dev)[None] < lens_d[:, None]
        assert (got[~keep] == 0).all(), f"{what}: masked rows are not 0"
    err = (got.double() - ref).abs()
    bound = _ln_bound(ref, xhat, sd, vmax, w.double(), bb.double(), dim) + (U32 * w.double().abs() * vmax / sd if res else 0.0)
    worst = (err / bound)[keep].max().item() if keep.any() else 0.0
    assert worst <= 1.0, f"{what}: error {err[keep].max().item():.3e} is {worst:.2f}x the bound"
    return worst


LN_DIMS = (8, 64, 128, 160, 256, 1000, 1024, 1280, 2048)


@pytest.mark.parametrize("dim", LN_DIMS)
def test_layernorm_layouts(dim):
    """Dense; residual + sum_out; the T2U's halo-3 layout with the padding mask over lengths 0, 1 and T; the adaptor's
    pooled layout (in halo 0 -> out halo 4, out_rows != T + 8) with residual + sum_out."""
    T = 37
    _ln_case(dim, 2, T)
    _ln_case(dim, 3, T, res=True)
    _ln_case(dim, 3, T, in_halo=3, out_halo=3, lens=[T, 1, 0], mask=True)
    _ln_case(dim, 3, T, in_halo=3, out_halo=3, lens=[T, 1, 0], mask=False, res=True)
    _ln_case(dim, 2, T, in_halo=0, out_halo=4, out_rows=T + 11, res=True)


@pytest.mark.parametrize("B,T", [(1, 4095), (3, 1365), (1, 4096), (4, 1024), (1, 4097), (17, 241)])
def test_layernorm_rows_straddle_block_switch(B, T):
    """sb_layernorm packs 2 rows per CTA below 4096 rows and 8 from 4096 on."""
    _ln_case(1024, B, T)
    _ln_case(1024, B, T, in_halo=2, out_halo=2, lens=[T] + [max(0, T - 100 * i) for i in range(1, B)], mask=True, res=True)


@pytest.mark.parametrize("ratio", [0, 10, 100, 300, 1000])
def test_layernorm_offset_inputs(ratio):
    """x = c + N(0, 1) with c / sd up to 1e3 (at 1e3 an fp16 step is half the spread, but the reference reads the same
    fp16 values): the two-pass statistics keep the error inside the bound."""
    for dim in (256, 1024, 2048):
        _ln_case(dim, 2, 33, offset=float(ratio))
        _ln_case(dim, 2, 33, offset=float(ratio), res=True, in_halo=1, out_halo=1)


@pytest.mark.parametrize("dim", [12, 2056])
def test_layernorm_unsupported_dim(dim):
    """dim not a multiple of 8, or above 2048: SB_ENOSUP, nothing launched, nothing written."""
    lib = _lib()
    x = torch.zeros(4, dim, dtype=torch.float16, device=dev)
    y = torch.full_like(x, SENT)
    w = torch.ones(dim, device=dev)
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    for fn in ("layernorm", "splitk"):
        if fn == "layernorm":
            rc = lib.sb_layernorm(x.data_ptr(), None, y.data_ptr(), None, w.data_ptr(), w.data_ptr(), dim, 1, 4, 4, 0, 4, 0,
                                  None, 0, _stream())
        else:
            part = torch.zeros(1, 4, dim, device=dev)
            rc = lib.sb_splitk_reduce_ln(part.data_ptr(), 1, 4, 4, dim, None, x.data_ptr(), w.data_ptr(), w.data_ptr(),
                                         y.data_ptr(), _stream())
        assert rc == SB_ENOSUP, (fn, rc)
    torch.cuda.synchronize()
    assert lib.sb_launch_count() == n0
    assert (_bits(y) == SENT_BITS).all() and (x == 0).all()


@pytest.mark.parametrize("dim", [256, 1024, 2048])
@pytest.mark.parametrize("splits", [1, 2, 3, 4, 5, 7, 8, 12, 13, 16])
def test_splitk_reduce_ln(splits, dim):
    """x += bias + partial[0] + partial[1] + ... must equal that fp32 sum taken left to right and rounded once, bit for
    bit (every chunk size of the kernel's gather: 8, 4, 1); h = LN(x) meets the LayerNorm bound (_ln_bound) on the
    rounded x.  Rows between `rows` and slice_rows in each slice hold NaN, and the rows after `rows` are untouched."""
    lib = _lib()
    rows, slice_rows = 37, 128
    g = torch.Generator(device=dev).manual_seed(splits * 31 + dim)
    for with_bias in (False, True):
        part = torch.full((splits, slice_rows, dim), math.nan, device=dev)
        part[:, :rows] = torch.randn(splits, rows, dim, device=dev, generator=g) / math.sqrt(splits)
        bias = torch.randn(dim, device=dev, generator=g) * 0.3 if with_bias else None
        x0 = torch.randn(rows + 2, dim, device=dev, generator=g).half()
        x0[rows:] = SENT
        w = torch.rand(dim, device=dev, generator=g) + 0.5
        bb = torch.randn(dim, device=dev, generator=g) * 0.2
        x = x0.clone()
        h = torch.full_like(x0, SENT)
        rc = lib.sb_splitk_reduce_ln(part.data_ptr(), splits, rows, slice_rows, dim, None if bias is None else bias.data_ptr(),
                                     x.data_ptr(), w.data_ptr(), bb.data_ptr(), h.data_ptr(), _stream())
        assert rc == SB_OK, lib.sb_last_error()
        acc = x0[:rows].float()
        if bias is not None:
            acc = acc + bias
        for z in range(splits):
            acc = acc + part[z, :rows]
        xe = acc.half()
        what = f"splits={splits} dim={dim} bias={with_bias}"
        assert torch.equal(_bits(x[:rows]), _bits(xe)), f"{what}: x"
        assert (_bits(x[rows:]) == SENT_BITS).all() and (_bits(h[rows:]) == SENT_BITS).all(), f"{what}: rows past `rows`"
        ref, xhat, sd, vmax = _ln_ref(xe.double(), w.double(), bb.double())
        err = (h[:rows].double() - ref).abs()
        worst = (err / _ln_bound(ref, xhat, sd, vmax, w.double(), bb.double(), dim)).max().item()
        assert worst <= 1.0, f"{what}: h error {err.max().item():.3e} is {worst:.2f}x the bound"


# ================================================================================================ sb_dwconv_ln_silu
def _dw_case(B, T, C, k, *, ratio=None, seed=0):
    """Causal depthwise conv (left pad k - 1) -> LayerNorm(C) -> SiLU against float64.  ratio: positive taps, in
    [0.5, 1.5) normalised to sum 1 per channel, and x = c + N(0, 1) with c = ratio * rms_c |w_c|, so that every channel
    of a full frame has mean ~c and sd ~|w_c|: the LayerNorm sees channel mean / sd ~ratio.  Returns the largest
    mean / sd of a frame and the worst error-to-bound ratio.

    Bound.  Each conv output a_c is an fp32 sum of k products (the kernels' order is sequential in the tap): |d a_c| <=
    k u A_c with A_c = sum_j |w_cj x_(t-j)c| (gamma bound).  The centred LayerNorm statistics of _ln_bound, with the conv error
    carried through (it moves x^_c by |d a_c| / sd directly and by at most max_c |d a_c| / sd through the mean):
    |d x^| <= u ((n max|a| + 2 k max A) / sd + (n / 2 + 8) |x^|), n = C / 32 + 21.  SiLU' is at most 1.1 and __expf
    adds ~1e-6 relative: |y - ref| <= 2^-11 |ref| + 1.1 (|w| |d x^| + u (|w x^| + |b|)) + 2e-6 |ref|."""
    lib = _lib()
    g = torch.Generator(device=dev).manual_seed(seed * 7919 + B * 131 + T * 17 + C * 3 + k)
    if ratio is None:
        w = (torch.randn(C, k, device=dev, generator=g) * 0.2).half()
        x = torch.randn(B, T, C, device=dev, generator=g).half()
    else:
        wt = torch.rand(C, k, device=dev, generator=g) + 0.5
        w = (wt / wt.sum(1, keepdim=True)).half()
        c = ratio * w.float().pow(2).sum(1).mean().sqrt().item()
        x = (c + torch.randn(B, T, C, device=dev, generator=g)).half()
    lw = torch.rand(C, device=dev, generator=g) + 0.5
    lb = torch.randn(C, device=dev, generator=g) * 0.2
    y = torch.full((B * T + 3, C), SENT, dtype=torch.float16, device=dev)

    def call(b0, nb, out):
        rc = lib.sb_dwconv_ln_silu(x[b0].data_ptr(), out.data_ptr(), w.data_ptr(), lw.data_ptr(), lb.data_ptr(), nb, T, C, k,
                                   _stream())
        assert rc == SB_OK, lib.sb_last_error()

    call(0, B, y)
    what = f"B={B} T={T} C={C} k={k} ratio={ratio}"
    assert (_bits(y[B * T:]) == SENT_BITS).all(), f"{what}: wrote past the output"
    xp = F.pad(x.double().transpose(1, 2), (k - 1, 0))
    a = F.conv1d(xp, w.double().view(C, 1, k), groups=C).transpose(1, 2)            # (B, T, C)
    A = F.conv1d(xp.abs(), w.double().abs().view(C, 1, k), groups=C).transpose(1, 2)
    mean = a.mean(-1, keepdim=True)
    sd = ((a - mean) ** 2).mean(-1, keepdim=True).add(1e-5).sqrt()
    xhat = (a - mean) / sd
    z = xhat * lw.double() + lb.double()
    ref = z * torch.sigmoid(z)
    n = C / 32 + 21
    dx = U32 * ((n * a.abs().amax(-1, keepdim=True) + 2 * k * A.amax(-1, keepdim=True)) / sd + (n / 2 + 8) * xhat.abs())
    bound = (2.0 ** -11 + 2e-6) * ref.abs() + 1.1 * (lw.double().abs() * dx + U32 * ((lw.double() * xhat).abs() + lb.double().abs()))
    got = y[:B * T].view(B, T, C)
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got.double() - ref).abs()
    worst = (err / bound).max().item()
    measured = (mean.abs() / sd).max().item()
    assert worst <= 1.0, f"{what}: error {err.max().item():.3e} is {worst:.2f}x the bound (channel mean / sd {measured:.0f})"
    for b in range(B):
        one = torch.full((T, C), SENT, dtype=torch.float16, device=dev)
        call(b, 1, one)
        assert torch.equal(_bits(one), _bits(got[b])), f"{what}: sequence {b} alone differs from the batch"
    again = torch.full_like(y, SENT)
    call(0, B, again)
    assert torch.equal(_bits(again), _bits(y)), f"{what}: repeated call differs"
    return measured, worst


DW_T = (1, 8, 9, 15, 31, 32, 33, 63, 64, 65, 499, 1000)
DW_RATIOS = (0.0, 5.0, 20.0, 40.0, 100.0, 300.0)  # channel mean / sd of the conv output, reached through offset inputs


def _dw_offset_sweep(C, k):
    for target in DW_RATIOS:
        measured, _ = _dw_case(2, 70, C, k, ratio=target)
        assert target == 0 or measured > 0.5 * target, (target, measured)  # the sweep reaches the ratio it names


def _dw_sweep(C, k=31):
    for T in DW_T:
        _dw_case(3, T, C, k)
    _dw_case(40, 33, C, k)
    _dw_offset_sweep(C, k)


@pytest.mark.parametrize("C", [64, 128, 256, 512, 1024])
def test_dwconv_tile_kernel(C):
    """k = 31, C % 64 == 0: the 32-frame tile kernel, with C / 64 warps combining the LayerNorm statistics.  It keeps
    var = E[a^2] - mean^2 up to channel mean / sd 8 (ratios 0 and 5 here) and combines per-warp centred sums of squares
    beyond (20 to 300): E[a^2] - mean^2 in fp32 misses the bound from mean / sd ~100 on."""
    _dw_sweep(C)


@pytest.mark.parametrize("C", [8, 72, 200])
def test_dwconv_fixed31_kernel(C):
    """k = 31 with C % 64 != 0: the 8-frame fixed-31 kernel."""
    _dw_sweep(C)


@pytest.mark.parametrize("k", [1, 3, 15, 32])
def test_dwconv_generic_kernel(k):
    """Any other k: the generic kernel (taps transposed into shared memory)."""
    for C in (72, 256):
        _dw_sweep(C, k)


def _dw_fixed31_wide():
    for C in (256, 1024):
        _dw_sweep(C)
    torch.cuda.synchronize()


def test_dwconv_fixed31_kernel_at_encoder_widths():
    """SB_DWCONV_TILE=0 (read once per process) sends C = 256 and 1024 to the fixed-31 kernel: in a child process."""
    _child("_dw_fixed31_wide", "SB_DWCONV_TILE", "0")
