"""The speech-output kernels between the text decoder and the waveform, called through the C-ABI and checked against
float64 references built from the kernels' own fp16 inputs.

sb_hifigan_resblock (csrc/resblock.cu): the fused ResBlock of the 16- and 32-channel generator stages, at the
production (kernel, dilations) pairs and at the geometry edges the entry accepts (k = 1; hk * d = 30 with H = 105; hk * d
= 32, the guard rows), over lengths that straddle its 640-row tiles, ragged batches with idle tiles, both halos of the
production layout (800 / 1600 rows at 79 200 / 158 400 rows) and rows_per_seq > T + 2 halo.
The ConvTranspose1d -> 3-tap GEMM repack (engine.conv_transpose_taps), in float64 on the CPU and through sb_gemm.
sb_conv_post_tanh, sb_vocoder_embed (csrc/vocoder.cu); sb_upsample_add, sb_durations, sb_unit_argmax (csrc/nar.cu).

Inputs no kernel may read (halo rows, rows past a sequence's length, padding columns) hold NaN (or +inf), and every
output element outside the written region holds a sentinel that must survive bit for bit.

The ResBlock bound.  The reference runs hifigan.py's ResBlock (xt = c2(lrelu(c1(lrelu(x)))); x = xt + x, three times,
then out = (x + res2) * gamma, out2 = lrelu(out)) in float64 on each sequence alone, zero padded past its length, and
rounds to fp16 where the kernel does: as = fp16(lrelu(x)), ts = fp16(lrelu(conv1 + b1)), xs = fp16(conv2 + b2 + xs),
as = fp16(lrelu(unrounded xs)), out / out2 from the fp16 xs.  Alongside each reference value v it carries E, a bound on
|kernel - v| before the rounding: each conv adds the fp32 accumulation error gamma_n (sum |w| |a| + |b|) (n = k C + 32,
unit 2^-23: tensor-core sums may truncate) and propagates the incoming E through |W| (the elementwise form of the
||W||_inf propagation).  A rounding maps the interval [v - E, v + E] through fp16 (and lrelu, both monotone), so the
rounded values differ by at most max(|h(v +- E) - h(v)|): zero where the interval holds no rounding boundary, one fp16
step where it does.  The bound is rigorous, and an output error is either 0 or at least one fp16 step, so it has no slack.
Weights: folded weight-norm convs drawn as N(0, 1/(k C)) have ||W||_inf ~ 0.8 sqrt(k C) = 5 to 15, and a worst-case
bound multiplies by that at each of the six convs: 10^4 to 10^7 fp16 steps, which rejects nothing.  So each output
channel here reads two dominant taps of +-0.3 to 0.45 at random (tap, channel) positions plus dense N(0, s^2) weights
with sum |w| ~ 0.15 on every other position: ||W||_inf ~ 1, activations stay O(1), and every tap and channel of the
kernel's fragments carries weight.
Negative controls: the same bound rejects the kernel's output against references with one tap of a conv shifted by one
row, the dilations of pairs 1 and 2 swapped, conv2's bias dropped, and the receptive field cut at H - 1 rows from a tile's
valid rows (test_resblock_bound_rejects_wrong_references).  The controls use dominant taps at tap 0 with positive inputs
so that a tile's first valid row depends on the row H before it with gain ~0.7^6.

The other bounds are derived where they are used; u = 2^-24 is the fp32 unit roundoff."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from seamless_communication_b200.engine import conv_transpose_taps

gpu = pytest.mark.gpu
dev = "cuda"
SB_OK, SB_EINVAL, SB_ENOSUP = 0, -1, -3  # include/seamless_b200.h
U32 = 2.0 ** -24          # fp32 unit roundoff
U_TC = 2.0 ** -23         # tensor-core fp32 accumulation (alignment / truncation): twice the round-to-nearest unit
SENT = -777.0             # exact in fp16 and fp32; no kernel computes it from these inputs
SENT_BITS = torch.tensor(SENT, dtype=torch.float16).view(torch.int16).item()
INT32_MAX = 2 ** 31 - 1
RB_ROWS = 640             # resblock.cu: time rows per tile (valid rows plus both receptive-field halves)


def _lib():
    from seamless_communication_b200 import _lib as L
    return L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(torch.int16)


def _gamma(n, unit):
    return n * unit / (1 - n * unit)


# ================================================================================================ sb_hifigan_resblock
def _H(k, dil):
    """Receptive-field half width of the whole ResBlock: three convs1 (dilation d) and three convs2 (dilation 1)."""
    return (k - 1) // 2 * (sum(dil) + 3)


def _h(z):
    """fp16 rounding as float64 (monotone; exact round-to-nearest on fp32 values)."""
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


def _conv(a, W, b, d):
    k = W.shape[2]
    return F.conv1d(a, W, b, padding=(k - 1) // 2 * d, dilation=d)


def _conv_bound(a, Ea, W, b, d):
    """'same' conv of the reference a (1, C, L) with the incoming bound Ea: (value, bound on the kernel's fp32 value).
    Propagated: |W| * Ea.  Local: gamma_n (|W| * (|a| + Ea) + |b|), n = k C + 32 terms of the mma chain (16-term
    blocks summed with the accumulator, the bias and the residual added after it)."""
    n = W.shape[2] * W.shape[1] + 32
    Wa = W.abs()
    v = _conv(a, W, b, d)
    E = _conv(Ea, Wa, None, d) + _gamma(n, U_TC) * _conv(a.abs() + Ea, Wa, b.abs(), d)
    return v, E


def _rb_chain(x, P, dil, slope, defect=None):
    """float64 ResBlock of one sequence x (1, C, L) (fp16 values) at the kernel's rounding points -> (xs, bound).
    defect: None, or one of the negative controls' wrong references ("tap", "bias")."""
    a32 = x.float()
    a = torch.where(a32 > 0, a32, a32 * slope).half().double()  # the kernel's own fp32 lrelu, rounded once: exact
    Ea = torch.zeros_like(a)
    xs, Ex = x, torch.zeros_like(x)
    for i in range(3):
        v, E = _conv_bound(a, Ea, P["w1"][i], P["b1"][i], dil[i])
        if defect == "tap" and i == 0:  # tap 0 of the first conv reads one row too late
            Wt = torch.zeros_like(P["w1"][0])
            Wt[:, :, 0] = P["w1"][0][:, :, 0]
            v = v - _conv(a, Wt, None, dil[0]) + _conv(F.pad(a[..., 1:], (0, 1)), Wt, None, dil[0])
        t, Et = _rnd_lrelu(v, E, slope)
        b2 = torch.zeros_like(P["b2"][i]) if defect == "bias" and i == 0 else P["b2"][i]
        v2, E2 = _conv_bound(t, Et, P["w2"][i], b2, 1)
        v2 = v2 + xs
        E2 = E2 + Ex
        E2 = E2 + U32 * (v2.abs() + E2)  # the fp32 residual add
        xs, Ex_new = _rnd(v2, E2)
        a, Ea = _rnd_lrelu(v2, E2, slope)
        Ex = Ex_new
    return xs, Ex


def _rb_out(xs, Ex, r2, gamma, s2):
    """out = fp16((xs + res2) gamma), out2 = fp16(lrelu(that fp32 value, s2)): fp32 add and product, u each."""
    pre = (xs + r2) * gamma
    Ep = abs(gamma) * (Ex + U32 * (xs.abs() + Ex + r2.abs()))
    Ep = Ep + U32 * (pre.abs() + Ep)
    out, Eo = _rnd(pre, Ep)
    out2, Eo2 = _rnd_lrelu(pre, Ep, s2)
    return out, Eo, out2, Eo2


def _rb_ref(x_seq, r2_seq, P, k, dil, slope, gamma, s2, defect=None, tile=None):
    """Reference and bound of one sequence: x_seq / r2_seq (L, C) fp16 (r2 None: 0).  tile = (TT, Hc): each tile of TT
    valid rows sees only Hc rows of context either side (the receptive-field-cut control)."""
    x = x_seq.double().t()[None]
    r2 = torch.zeros_like(x) if r2_seq is None else r2_seq.double().t()[None]
    if tile is None:
        xs, Ex = _rb_chain(x, P, dil if defect != "dil" else (dil[0], dil[2], dil[1]), slope, defect)
    else:
        TT, Hc = tile
        L = x.shape[2]
        xs, Ex = torch.empty_like(x), torch.empty_like(x)
        for t0 in range(0, L, TT):
            w0, w1 = max(0, t0 - Hc), min(L, t0 + TT + Hc)
            a, e = _rb_chain(x[..., w0:w1], P, dil, slope)
            t1 = min(L, t0 + TT)
            xs[..., t0:t1], Ex[..., t0:t1] = a[..., t0 - w0:t1 - w0], e[..., t0 - w0:t1 - w0]
    out = _rb_out(xs, Ex, r2, gamma, s2)
    return tuple(o[0].t() for o in out)


def _ratio(got, ref, E):
    """max |got - ref| / E, with an error where E = 0 counted as infinite."""
    err = (got.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / E)
    return r.max().item() if r.numel() else 0.0


def _rb_weights(C, k, g, device, control=False):
    """Six convs (C, C, k) float64 holding fp16 values, fp32 biases.  Each output channel: two dominant weights of
    +-U(0.3, 0.45) at random (tap, input channel) positions, and N(0, s^2) elsewhere with s = 0.15 / (0.8 k C), so that
    sum |w| over a row is ~1.  control: one dominant +0.7 at tap 0 per output channel, positive biases."""
    P = {n: [] for n in ("w1", "b1", "w2", "b2")}
    s = 0.15 / (0.8 * k * C)
    for _ in range(3):
        for wn, bn in (("w1", "b1"), ("w2", "b2")):
            W = torch.randn(C, C, k, generator=g, device=device) * s
            co = torch.arange(C, device=device)
            if control:
                W[co, torch.randperm(C, generator=g, device=device), 0] = 0.7
                b = torch.rand(C, generator=g, device=device) * 0.2
            else:
                for _m in range(2):
                    ci = torch.randperm(C, generator=g, device=device)
                    tap = torch.randint(0, k, (C,), generator=g, device=device)
                    sign = torch.randint(0, 2, (C,), generator=g, device=device) * 2 - 1
                    W[co, ci, tap] += sign * (0.3 + 0.15 * torch.rand(C, generator=g, device=device))
                b = (torch.rand(C, generator=g, device=device) - 0.5) * 0.6
            P[wn].append(W.half().double())
            P[bn].append(b.float().double())
    return P


def _rb_kernel_weights(P):
    """Conv layout of sb_gemm / resblock.cu: (C, k * C) fp16 with w[co][tap * C + ci]; fp32 biases."""
    C, _, k = P["w1"][0].shape
    out = {}
    for n in ("w1", "w2"):
        out[n] = [W.permute(0, 2, 1).reshape(C, k * C).half().contiguous() for W in P[n]]
    for n in ("b1", "b2"):
        out[n] = [b.float().contiguous() for b in P[n]]
    return out


def _rb_call(KW, x, r2, out, out2, C, k, dil, B, T, rows, halo, lens, gamma, s2, slope=0.1):
    from seamless_communication_b200 import _lib as L
    d = L.ResblockDesc()
    d.x, d.res2, d.out = x.data_ptr(), None if r2 is None else r2.data_ptr(), out.data_ptr()
    d.out2 = None if out2 is None else out2.data_ptr()
    for i in range(3):
        d.w1[i] = None if KW["w1"][i] is None else KW["w1"][i].data_ptr()
        d.b1[i] = KW["b1"][i].data_ptr()
        d.w2[i], d.b2[i] = KW["w2"][i].data_ptr(), KW["b2"][i].data_ptr()
        d.dilation[i] = dil[i]
    d.channels, d.kernel_size, d.batch, d.T, d.rows_per_seq, d.halo = C, k, B, T, rows, halo
    d.slope, d.gamma, d.out2_slope = slope, gamma, s2
    d.lens = None if lens is None else lens.data_ptr()
    return _lib().sb_hifigan_resblock(ctypes.byref(d), _stream())


def _rb_inputs(C, T, lens, halo, tail, g, control=False):
    B = len(lens)
    rows = T + 2 * halo + tail
    if control:
        x = (torch.rand(B, rows, C, device=dev, generator=g) + 0.25).half()
    else:
        x = torch.randn(B, rows, C, device=dev, generator=g).half()
    r2 = torch.randn(B, rows, C, device=dev, generator=g).half()
    for t in (x, r2):  # nothing outside each sequence's rows [halo, halo + lens[b]) is read
        t[:, :halo] = math.nan
        for b in range(B):
            t[b, halo + lens[b]:] = math.nan
    return x, r2, rows


def _rb_case(C, k, dil, T, lens, *, halo=0, tail=0, res2=False, gamma=1.0, out2=False, s2=0.1, seed=0, checks=True):
    """One batched sb_hifigan_resblock call against the float64 reference and bound; with checks, also: each sequence
    alone (T = lens[b]) equals the batch bit for bit, a permuted batch permutes the outputs bit for bit, and a repeated
    call is bit-identical."""
    B = len(lens)
    g = torch.Generator(device=dev).manual_seed(seed * 7919 + C * 131 + k * 17 + T + halo)
    P = _rb_weights(C, k, g, dev)
    KW = _rb_kernel_weights(P)
    x, r2, rows = _rb_inputs(C, T, lens, halo, tail, g)
    r2 = r2 if res2 else None
    gamma = float(torch.tensor(gamma, dtype=torch.float32))  # the kernel multiplies by the fp32 gamma
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)

    def run(xx, rr, ll, nb, TT, rw):
        o = torch.full((nb, rw, C), SENT, dtype=torch.float16, device=dev)
        o2 = torch.full_like(o, SENT) if out2 else None
        rc = _rb_call(KW, xx, rr, o, o2, C, k, dil, nb, TT, rw, halo, ll, gamma, s2)
        assert rc == SB_OK, _lib().sb_last_error()
        return o, o2

    what = f"C={C} k={k} dil={dil} T={T} lens={lens} halo={halo} tail={tail} res2={res2} gamma={gamma:.3f} out2={out2}"
    n0 = _lib().sb_launch_count()
    out, o2 = run(x, r2, lens_d, B, T, rows)
    assert _lib().sb_launch_count() == n0 + 1
    worst = 0.0
    for b in range(B):
        L = lens[b]
        for o, name in ((out, "out"), (o2, "out2")):
            if o is None:
                continue
            assert (o[b, :halo] == 0).all() and (o[b, halo + T:halo + T + halo] == 0).all(), f"{what} b={b}: {name} halo rows"
            assert (o[b, halo + L:halo + T] == 0).all(), f"{what} b={b}: {name} rows past lens are not 0"
            assert (_bits(o[b, T + 2 * halo:]) == SENT_BITS).all(), f"{what} b={b}: {name} wrote past the halo"
        if L == 0:
            continue
        ref, E, ref2, E2 = _rb_ref(x[b, halo:halo + L], None if r2 is None else r2[b, halo:halo + L], P, k, dil, 0.1,
                                   gamma, s2)
        r = _ratio(out[b, halo:halo + L], ref, E)
        assert r <= 1.0, f"{what} b={b}: out error is {r:.2f}x the bound"
        worst = max(worst, r)
        if out2:
            r = _ratio(o2[b, halo:halo + L], ref2, E2)
            assert r <= 1.0, f"{what} b={b}: out2 error is {r:.2f}x the bound"
    if not checks:
        return worst
    for b in range(B):  # alone, T = lens[b], the same halo and no tail
        L = lens[b]
        if L == 0:
            continue
        xa = torch.full((1, L + 2 * halo, C), math.nan, dtype=torch.float16, device=dev)
        xa[0, halo:halo + L] = x[b, halo:halo + L]
        ra = None
        if r2 is not None:
            ra = torch.full_like(xa, math.nan)
            ra[0, halo:halo + L] = r2[b, halo:halo + L]
        oa, oa2 = run(xa, ra, None, 1, L, L + 2 * halo)
        assert torch.equal(_bits(oa[0, halo:halo + L]), _bits(out[b, halo:halo + L])), f"{what}: sequence {b} alone differs"
        if out2:
            assert torch.equal(_bits(oa2[0, halo:halo + L]), _bits(o2[b, halo:halo + L])), f"{what}: out2 {b} alone differs"
    perm = list(range(B))[::-1]
    op, op2 = run(x[perm].contiguous(), None if r2 is None else r2[perm].contiguous(), lens_d[perm].contiguous(), B, T, rows)
    assert torch.equal(_bits(op), _bits(out[perm])), f"{what}: a permuted batch does not permute the outputs"
    if out2:
        assert torch.equal(_bits(op2), _bits(o2[perm])), f"{what}: out2 of a permuted batch"
    again, again2 = run(x, r2, lens_d, B, T, rows)
    assert torch.equal(_bits(again), _bits(out)) and (not out2 or torch.equal(_bits(again2), _bits(o2))), \
        f"{what}: repeated call differs"
    return worst


def _rb_T_list(k, dil):
    H = _H(k, dil)
    TT = RB_ROWS - 2 * H
    return sorted({t for t in (1, H, TT - 1, TT, TT + 1, 2 * TT + 1, 3 * TT) if t >= 1}), TT


def _rb_lens(T, TT):
    """Full, 0, 1, inside a tile and on a tile boundary, in one batch: tiles past a short row are idle."""
    mid = TT // 2 + 7 if T > TT // 2 + 7 else T // 2 + 1
    edge = TT if T > TT else max(1, T - 1)
    return [T, 0, 1, mid, edge]


# halo, tail (rows_per_seq - T - 2 halo), res2, gamma, out2, out2_slope: cycled over the lengths of each geometry
RB_VARIANTS = [(0, 0, False, 1.0, False, 0.1), (7, 0, True, 1 / 3, True, 0.01), (3, 5, True, 1.0, False, 0.1),
               (25, 3, False, 1 / 3, True, 0.1), (0, 9, True, 1 / 3, True, 0.1), (11, 0, False, 1.0, True, 0.01),
               (1, 2, True, 1.0, True, 0.1)]


def _rb_geometry_sweep(C, k, dil):
    Ts, TT = _rb_T_list(k, dil)
    for i, T in enumerate(Ts):
        halo, tail, res2, gamma, out2, s2 = RB_VARIANTS[(i + C + k) % len(RB_VARIANTS)]
        _rb_case(C, k, dil, T, _rb_lens(T, TT), halo=halo, tail=tail, res2=res2, gamma=gamma, out2=out2, s2=s2)


@gpu
@pytest.mark.parametrize("k", [3, 7, 11])
@pytest.mark.parametrize("C", [16, 32])
def test_resblock_production_pairs(C, k):
    """The production (k, dilations (1, 3, 5)) pairs: H = 12 / 36 / 60, 616 / 568 / 520 valid rows per tile; T = 1, H,
    TT - 1, TT, TT + 1, 2 TT + 1, 3 TT with ragged lengths, halos 0 to 25, tails, res2, gamma, out2 in rotation."""
    _rb_geometry_sweep(C, k, (1, 3, 5))


@gpu
@pytest.mark.parametrize("k,dil", [(1, (1, 1, 1)), (11, (6, 6, 6)), (3, (32, 32, 32))])
@pytest.mark.parametrize("C", [16, 32])
def test_resblock_geometry_edges(C, k, dil):
    """k = 1 (H = 0, 640 valid rows per tile); k = 11 with dilation 6 (tap offset 30, H = 105); k = 3 with dilation 32
    (tap offset = the 32 guard rows, H = 99)."""
    _rb_geometry_sweep(C, k, dil)


@gpu
@pytest.mark.parametrize("C,U", [(32, 495), (16, 495)])
def test_resblock_production_length(C, U):
    """The bench's 9.9 s rows: U = 495 units give T = 79 200 rows at 32 channels and 158 400 at 16, with the production
    halos 800 / 1600; one full row and one ending inside a tile, through each of the three ResBlocks."""
    rate = 160 if C == 32 else 320
    T, halo = U * rate, 5 * rate
    for i, k in enumerate((3, 7, 11)):
        _rb_case(C, k, (1, 3, 5), T, [T, T - 12345], halo=halo, res2=i > 0, gamma=1 / 3 if k == 11 else 1.0, out2=k == 11,
                 s2=0.1 if C == 32 else 0.01, checks=(k == 11))


@gpu
@pytest.mark.parametrize("C,k", [(16, 3), (32, 11)])
def test_resblock_bound_rejects_wrong_references(C, k):
    """Negative controls: the kernel's output meets the bound against the right reference and fails it against each
    wrong one (a tap shifted by one row, dilations of pairs 1 and 2 swapped, conv2's bias dropped, the receptive field
    cut at H - 1 rows from a tile's valid rows)."""
    dil = (1, 3, 5)
    H = _H(k, dil)
    TT = RB_ROWS - 2 * H
    T = 2 * TT + 1
    lens = [T, TT + 5]
    g = torch.Generator(device=dev).manual_seed(C * 17 + k)
    P = _rb_weights(C, k, g, dev, control=True)
    KW = _rb_kernel_weights(P)
    x, _, rows = _rb_inputs(C, T, lens, 0, 0, g, control=True)
    out = torch.full((2, rows, C), SENT, dtype=torch.float16, device=dev)
    rc = _rb_call(KW, x, None, out, None, C, k, dil, 2, T, rows, 0, torch.tensor(lens, dtype=torch.int32, device=dev),
                  1.0, 0.1)
    assert rc == SB_OK, _lib().sb_last_error()
    for b, L in enumerate(lens):
        got = out[b, :L]
        ref, E, _, _ = _rb_ref(x[b, :L], None, P, k, dil, 0.1, 1.0, 0.1)
        assert _ratio(got, ref, E) <= 1.0, f"b={b}: the right reference fails the bound"
        for defect in ("tap", "dil", "bias", "cut"):
            if defect == "cut":
                wref, wE, _, _ = _rb_ref(x[b, :L], None, P, k, dil, 0.1, 1.0, 0.1, tile=(TT, H - 1))
            else:
                wref, wE, _, _ = _rb_ref(x[b, :L], None, P, k, dil, 0.1, 1.0, 0.1, defect=defect)
            r = _ratio(got, wref, wE)
            assert r > 1.0, f"b={b}: the bound accepts the wrong reference {defect!r} ({r:.2f}x)"


@gpu
@pytest.mark.parametrize("what", ["C8", "C24", "C64", "k2", "k13", "k3d33", "k11d7", "rows", "null_w"])
def test_resblock_refusals(what):
    """Shapes the kernel cannot run return SB_EINVAL before anything is launched, and nothing is written."""
    C = {"C8": 8, "C24": 24, "C64": 64}.get(what, 16)
    k = {"k2": 2, "k13": 13, "k3d33": 3, "k11d7": 11}.get(what, 3)
    dil = {"k3d33": (1, 33, 1), "k11d7": (1, 3, 7)}.get(what, (1, 3, 5))
    T, halo = 50, 4
    rows = T + 2 * halo - (1 if what == "rows" else 0)
    g = torch.Generator(device=dev).manual_seed(1)
    KW = _rb_kernel_weights(_rb_weights(C, max(k, 1), g, dev))
    if what == "null_w":
        KW["w1"][1] = None
    x = torch.zeros(2, T + 2 * halo, C, dtype=torch.float16, device=dev)
    out = torch.full_like(x, SENT)
    torch.cuda.synchronize()
    n0 = _lib().sb_launch_count()
    rc = _rb_call(KW, x, None, out, None, C, k, dil, 2, T, rows, halo, None, 1.0, 0.1)
    torch.cuda.synchronize()
    assert rc == SB_EINVAL, (what, rc)
    assert _lib().sb_launch_count() == n0
    assert (_bits(out) == SENT_BITS).all()


# ================================================================================================ ConvTranspose taps
def _taps_apply(x, wt, u, cout):
    """The packed taps as the GEMM applies them: a zero-padded 3-tap conv at the input rate, phases interleaved.
    x (cin, T) -> (cout, T u)."""
    cin, T = x.shape
    y = F.conv1d(x[None], wt.view(u * cout, 3, cin).permute(0, 2, 1), padding=1)[0]  # (u cout, T)
    return y.view(u, cout, T).permute(1, 2, 0).reshape(cout, T * u)


def test_conv_transpose_taps_match_conv_transpose1d():
    """Every (u <= 6, u <= k <= 3u) with k - u even: the packed taps equal F.conv_transpose1d(stride u, padding
    (k - u) / 2) in float64 (error 1e-12: a few float64 roundings of O(10) sums).  This covers the shipped cards'
    (5, 11), (4, 8), (2, 4).  Every other pair (k - u odd, k < u, k > 3u) raises ValueError."""
    g = torch.Generator().manual_seed(0)
    cin, cout, T = 6, 5, 9
    for u in range(1, 7):
        for k in range(1, 3 * u + 4):
            cw = torch.randn(cin, cout, k, generator=g, dtype=torch.float64)
            if (k - u) % 2 or not u <= k <= 3 * u:
                with pytest.raises(ValueError):
                    conv_transpose_taps(cw, u, k)
                continue
            x = torch.randn(cin, T, generator=g, dtype=torch.float64)
            ref = F.conv_transpose1d(x[None], cw, stride=u, padding=(k - u) // 2)[0]
            got = _taps_apply(x, conv_transpose_taps(cw, u, k), u, cout)
            assert got.shape == ref.shape == (cout, T * u), (u, k)
            assert (got - ref).abs().max().item() < 1e-12, (u, k)


@pytest.mark.parametrize("u,k", [(4, 16), (2, 5), (3, 2), (1, 4)])
def test_conv_transpose_taps_refuses_unrepresentable(u, k):
    """(4, 16) would drop taps 0, 1, 14 and 15; (2, 5) gives T u + 1 samples; (3, 2) needs negative padding; (1, 4)
    is even k - u.  None of them is a 3-tap conv: ValueError."""
    with pytest.raises(ValueError):
        conv_transpose_taps(torch.zeros(4, 3, k), u, k)


BASE_UPS = [(512, 5, 11), (256, 4, 8), (128, 4, 8), (64, 2, 4), (32, 2, 4)]  # (cin, u, k): base vocoder, cout = cin / 2


@gpu
@pytest.mark.parametrize("cin,u,k", BASE_UPS)
def test_conv_transpose_gemm_matches_conv_transpose1d(cin, u, k):
    """The packed fp16 taps through ops.gemm(taps=3, out, out2 = lrelu(out, 0.1)) in the engine's layout: a ragged batch
    masked at the input rate, halo 5, NaN in the rows the GEMM never reads (the outermost halo rows but one).  Against
    the float64 conv_transpose1d of each row alone: |err| <= gamma_{3 cin + 1} (sum |x| |w| + |b|) (unit 2^-23) plus
    the fp16 rounding of out (2^-11 |.|); out2 is lrelu of out's fp32 value or of its fp16 value: one more 2^-11
    rounding.  Rows past u lens[b] are exactly 0."""
    from seamless_communication_b200 import ops
    cout, T, PH = cin // 2, 150, 5
    lens = [T, 1, 0, 77]
    B, Tp = len(lens), T + 2 * PH
    g = torch.Generator(device=dev).manual_seed(cin + u + k)
    cw = (torch.randn(cin, cout, k, device=dev, generator=g) / math.sqrt(cin * k / u)).half().double()
    bias = torch.randn(cout, device=dev, generator=g).float() * 0.3
    wt = conv_transpose_taps(cw.cpu(), u, k).to(dev).half().contiguous()
    bw = bias.repeat(u).contiguous()
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    act = ops.Seq(B, T, cin, PH, Tp, lens=lens_d, zero=True)
    xv = act.buf.view(B, Tp, cin)
    for b in range(B):
        xv[b, PH:PH + lens[b]] = torch.randn(lens[b], cin, device=dev, generator=g).half()
    act.buf[:PH - 1] = math.nan
    act.buf[B * Tp - PH + 1:] = math.nan
    up_raw = ops.Seq(B, T, u * cout, PH, Tp, lens=lens_d, zero="edges")
    up_act = ops.Seq(B, T, u * cout, PH, Tp, lens=lens_d, zero="edges")
    ops.gemm(act, wt, u * cout, bw, taps=3, out=up_raw, out2=up_act, out2_slope=0.1)
    raw = up_raw.buf.view(B, Tp * u, cout)
    ra = up_act.buf.view(B, Tp * u, cout)
    g_n = _gamma(3 * cin + 1, U_TC)
    for b in range(B):
        L = lens[b]
        got, got2 = raw[b, PH * u:(PH + T) * u], ra[b, PH * u:(PH + T) * u]
        assert (got[L * u:] == 0).all() and (got2[L * u:] == 0).all(), f"b={b}: rows past u lens are not 0"
        if L == 0:
            continue
        x = xv[b, PH:PH + L].double().t()[None]
        ref = (F.conv_transpose1d(x, cw, stride=u, padding=(k - u) // 2)[0] + bias.double()[:, None]).t()
        A = (F.conv_transpose1d(x.abs(), cw.abs(), stride=u, padding=(k - u) // 2)[0] + bias.double().abs()[:, None]).t()
        pre = g_n * A
        bound = pre + 2.0 ** -11 * (ref.abs() + pre) + 2.0 ** -25
        r = _ratio(got[:L * u], ref, bound)
        assert r <= 1.0, f"b={b}: out error is {r:.2f}x the bound"
        ref2 = _lrelu(ref, 0.1)
        bound2 = bound + 2.0 ** -11 * (ref2.abs() + bound) + U32 * ref.abs()
        r = _ratio(got2[:L * u], ref2, bound2)
        assert r <= 1.0, f"b={b}: out2 error is {r:.2f}x the bound"


# ================================================================================================ sb_conv_post_tanh
def _post_case(C, k, T, lens, halo, g):
    """wav[b][t] = tanh(bias + sum_{j,c} x[t + j - k/2][c] w[j][c]) for t < lens[b], 0 past it; columns past T keep
    the sentinel.  x: NaN outside the rows the kernel reads ([halo - k/2, halo + lens[b] + k/2)), zero halo / padding rows
    inside them.  Bound: the fp32 sum of k C + 1 terms, gamma_{k C + 1} (|bias| + sum |x w|) (tanh' <= 1), plus tanhf's
    2 ulp (2^-22 |.|)."""
    lib = _lib()
    B, hk = len(lens), k // 2
    rows = T + 2 * halo + 2
    x = torch.full((B, rows, C), math.nan, dtype=torch.float16, device=dev)
    for b in range(B):
        L = lens[b]
        x[b, halo - hk:halo + L + hk] = 0
        x[b, halo:halo + L] = torch.randn(L, C, device=dev, generator=g).half()
    w = (torch.randn(k, C, device=dev, generator=g) * 2 / math.sqrt(k * C)).half()
    bias = 0.1
    wav_ld = T + 5
    wav = torch.full((B, wav_ld), SENT, dtype=torch.float32, device=dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev)
    rc = lib.sb_conv_post_tanh(x.data_ptr(), rows, halo, T, lens_d.data_ptr(), C, B, w.data_ptr(), bias, k,
                               wav.data_ptr(), wav_ld, _stream())
    assert rc == SB_OK, lib.sb_last_error()
    what = f"C={C} k={k} T={T} lens={lens} halo={halo}"
    assert (wav[:, T:] == SENT).all(), f"{what}: wrote past T"
    w64 = w.double().t()[None]  # (1, C, k)
    for b in range(B):
        L = lens[b]
        assert (wav[b, L:T] == 0).all(), f"{what} b={b}: rows past lens are not 0"
        if L == 0:
            continue
        xs = x[b, halo - hk:halo + L + hk].double().t()[None]  # zero rows at both ends: the 'same' padding
        s = F.conv1d(xs, w64)[0, 0] + bias
        A = F.conv1d(xs.abs(), w64.abs())[0, 0] + abs(bias)
        ref = torch.tanh(s)
        bound = _gamma(k * C + 1, U32) * A + 2.0 ** -22 * ref.abs() + 1e-30
        r = _ratio(wav[b, :L], ref, bound)
        assert r <= 1.0, f"{what} b={b}: error is {r:.2f}x the bound"


@gpu
@pytest.mark.parametrize("k", [1, 3, 7])
@pytest.mark.parametrize("C", [8, 16, 32])
def test_conv_post_tanh(C, k):
    """T across the 256-row blocks, halo exactly k/2 and wider, lengths 0, 1 and T."""
    g = torch.Generator(device=dev).manual_seed(C * 10 + k)
    for T in (1, 255, 256, 257, 1000):
        for halo in (k // 2, k // 2 + 3):
            _post_case(C, k, T, [T, 0, 1, max(1, T // 2)], halo, g)


@gpu
@pytest.mark.parametrize("what", ["C12", "halo"])
def test_conv_post_tanh_refusals(what):
    """C not a multiple of 8, or a halo narrower than k/2: SB_ENOSUP, nothing launched, nothing written."""
    lib = _lib()
    C, k = (12, 7) if what == "C12" else (16, 7)
    halo = 3 if what == "C12" else 2
    x = torch.zeros(2, 20 + 2 * halo, C, dtype=torch.float16, device=dev)
    w = torch.zeros(k * C, dtype=torch.float16, device=dev)
    wav = torch.full((2, 20), SENT, dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    rc = lib.sb_conv_post_tanh(x.data_ptr(), 20 + 2 * halo, halo, 20, None, C, 2, w.data_ptr(), 0.0, k, wav.data_ptr(),
                               20, _stream())
    torch.cuda.synchronize()
    assert rc == SB_ENOSUP, rc
    assert lib.sb_launch_count() == n0
    assert (wav == SENT).all()


# ================================================================================================ sb_vocoder_embed
@gpu
@pytest.mark.parametrize("dims", [(256, 1280, 256), (32, 64, 32), (3, 5, 7)])
def test_vocoder_embed(dims):
    """x[b][u] = [lang[lang_idx[b]] | dict[units[b][u]] | spkr[spkr_idx[b]]] bit for bit: the base and tiny widths and odd
    ones, unit ids 0 and num_embeddings - 1, per-row language and speaker ids; halo rows keep the sentinel."""
    lib = _lib()
    ld, dd, sd = dims
    n_emb, n_lang, n_spkr, B, U, halo = 10000, 36, 200, 3, 37, 4
    g = torch.Generator(device=dev).manual_seed(sum(dims))
    dict_t = torch.randn(n_emb, dd, device=dev, generator=g).half()
    lang_t = torch.randn(n_lang, ld, device=dev, generator=g).half()
    spkr_t = torch.randn(n_spkr, sd, device=dev, generator=g).half()
    units = torch.randint(0, n_emb, (B, U), device=dev, generator=g, dtype=torch.int32)
    units[0, 0], units[1, -1], units[2, 5] = 0, n_emb - 1, n_emb - 1
    li = torch.tensor([0, n_lang - 1, 17], dtype=torch.int32, device=dev)
    si = torch.tensor([n_spkr - 1, 0, 45], dtype=torch.int32, device=dev)
    C = ld + dd + sd
    rows = U + 2 * halo
    x = torch.full((B, rows, C), SENT, dtype=torch.float16, device=dev)
    rc = lib.sb_vocoder_embed(units.data_ptr(), U, B, dict_t.data_ptr(), dd, lang_t.data_ptr(), ld, li.data_ptr(),
                              spkr_t.data_ptr(), sd, si.data_ptr(), x.data_ptr(), rows, halo, _stream())
    assert rc == SB_OK, lib.sb_last_error()
    for b in range(B):
        ref = torch.cat([lang_t[li[b].item()].expand(U, ld), dict_t[units[b].long()], spkr_t[si[b].item()].expand(U, sd)], 1)
        assert torch.equal(_bits(x[b, halo:halo + U]), _bits(ref)), f"row {b}"
    assert (_bits(x[:, :halo]) == SENT_BITS).all() and (_bits(x[:, halo + U:]) == SENT_BITS).all()


# ================================================================================================ sb_upsample_add
def _ulp16(v):
    """One fp16 step at |v| (2^-24 in the subnormal range)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def _durs(S, B, g):
    d = torch.randint(0, 4, (B, S), device=dev, generator=g, dtype=torch.int32)
    d[0, :min(3, S)] = 0                       # leading zeros
    if S > 4:
        d[0, S // 2:S // 2 + 2] = 0            # interior zeros
        d[0, -2:] = 0                          # trailing zeros
    d[B - 1] = 0                               # an all-zero row: total 0
    return d


def _upsample_case(S, dim, mode, U_kind, g):
    """mode "vocoder": pos / emb NULL, bit-exact against repeat_interleave.  mode "t2u": + alpha pos + emb scale, within one
    fp16 step of float64 x + (alpha pos + emb scale), plus the fp32 sum's 3 u (|x| + |alpha pos| + |emb scale|)."""
    lib = _lib()
    B, xh, yh = 3, 2, 3
    dur = _durs(S, B, g)
    tot = dur.sum(1).cpu()
    T = int(tot.max())
    U = {"exact": max(T, 1), "short": max(1, T - 17), "long": T + 21}[U_kind]
    if U_kind == "long" and U % 16 == 0:
        U += 1  # the last 16-row block of y is partial
    x = torch.randn(B, S + 2 * xh, dim, device=dev, generator=g).half()
    x[:, :xh] = math.nan
    x[:, xh + S:] = math.nan
    y = torch.full((B, U + 2 * yh + 1, dim), SENT, dtype=torch.float16, device=dev)
    out_lens = torch.full((B,), -1, dtype=torch.int32, device=dev)
    pos = alpha = emb = ids = None
    scale, ids_ld = 0.0, 0
    if mode == "t2u":
        pos = torch.randn(U, dim, device=dev, generator=g)
        alpha = torch.tensor([0.7], device=dev)
        emb = torch.randn(50, dim, device=dev, generator=g).half()
        ids_ld = U + 3
        ids = torch.randint(0, 50, (B, ids_ld), device=dev, generator=g, dtype=torch.int32)
        scale = 1.9
    rc = lib.sb_upsample_add(x.data_ptr(), S + 2 * xh, xh, S, dur.data_ptr(), y.data_ptr(), U + 2 * yh + 1, yh, U, B, dim,
                             None if pos is None else pos.data_ptr(), None if alpha is None else alpha.data_ptr(),
                             None if emb is None else emb.data_ptr(), None if ids is None else ids.data_ptr(), ids_ld,
                             scale, out_lens.data_ptr(), _stream())
    assert rc == SB_OK, lib.sb_last_error()
    what = f"S={S} dim={dim} mode={mode} U={U} (total {tot.tolist()})"
    assert out_lens.cpu().tolist() == tot.tolist(), f"{what}: out_lens"
    assert (_bits(y[:, :yh]) == SENT_BITS).all() and (_bits(y[:, yh + U:]) == SENT_BITS).all(), f"{what}: wrote outside"
    for b in range(B):
        n = min(int(tot[b]), U)
        got = y[b, yh:yh + U]
        assert (got[n:] == 0).all(), f"{what} b={b}: rows past the total are not exact zeros"
        src = torch.repeat_interleave(x[b, xh:xh + S], dur[b].long(), dim=0)[:n]
        if mode == "vocoder":
            assert torch.equal(_bits(got[:n]), _bits(src)), f"{what} b={b}"
            continue
        add = 0.7 * pos[:n].double() + emb[ids[b, :n].long()].double() * scale
        ref = src.double() + add
        bound = _ulp16(ref) + 3 * U32 * (src.double().abs() + add.abs() + (emb[ids[b, :n].long()].double() * scale).abs())
        r = _ratio(got[:n], ref, bound)
        assert r <= 1.0, f"{what} b={b}: error is {r:.2f}x one fp16 step"


@gpu
@pytest.mark.parametrize("S", [1, 255, 256, 257, 10240])
def test_upsample_add(S):
    """Across the 256-wide block scan up to the 40 KB shared-memory limit; dim 2, 6, 1024, 1026; U equal to, below
    (truncated rows, out_lens = the total) and above the largest total (zero rows), U not a multiple of 16."""
    g = torch.Generator(device=dev).manual_seed(S)
    for dim in (2, 6, 1024, 1026):
        for mode in ("vocoder", "t2u"):
            for U_kind in ("exact", "short", "long"):
                if S > 1000 and dim > 6 and U_kind != "long":
                    continue  # the long-U case already covers the widest rows at this length
                _upsample_case(S, dim, mode, U_kind, g)


@gpu
def test_upsample_add_refuses_long_sources():
    """S = 10 241 needs more than 40 KB of prefix sums: SB_ENOSUP, nothing launched."""
    lib = _lib()
    S = 10241
    x = torch.zeros(S, 2, dtype=torch.float16, device=dev)
    dur = torch.ones(S, dtype=torch.int32, device=dev)
    y = torch.full((S, 2), SENT, dtype=torch.float16, device=dev)
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    rc = lib.sb_upsample_add(x.data_ptr(), S, 0, S, dur.data_ptr(), y.data_ptr(), S, 0, S, 1, 2, None, None, None, None, 0,
                             0.0, None, _stream())
    torch.cuda.synchronize()
    assert rc == SB_ENOSUP, rc
    assert lib.sb_launch_count() == n0
    assert (_bits(y) == SENT_BITS).all()


# ================================================================================================ sb_durations
def _dur_case(dim, factor, B, S, lens, bias, spread, g):
    """dur = clamp(round_half_even((exp(h . w + b) - 1) factor), 1, INT32_MAX), 0 at s >= lens[b], compared exactly.
    An entry whose float64 pre-rounding value v lies within eps of a .5 boundary may round either way: logd is an fp32
    sum of 2 ceil(dim / 64) + 6 terms (a lane's products, 5 shuffle levels, the bias): |d logd| <= delta =
    gamma_n (sum |h w| + |b|); expf adds 2 ulp (2^-22); the subtraction and the product u each:
    eps = factor (e^logd (e^delta - 1 + 2^-22) + u (e^logd + 1)) + u |v|.  Returns how many such entries there were."""
    lib = _lib()
    halo = 2
    rows = S + 2 * halo
    h = torch.randn(B, rows, dim, device=dev, generator=g).half()
    h[:, :halo] = math.nan
    h[:, halo + S:] = math.nan
    w = (torch.randn(dim, device=dev, generator=g) * spread / math.sqrt(dim)).half()
    bias = float(torch.tensor(bias, dtype=torch.float32))
    lens_d = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    dur = torch.full((B, S), -5, dtype=torch.int32, device=dev)
    rc = lib.sb_durations(h.data_ptr(), rows, halo, w.data_ptr(), bias, dim, None if lens_d is None else lens_d.data_ptr(),
                          B, S, factor, dur.data_ptr(), _stream())
    assert rc == SB_OK, lib.sb_last_error()
    hd = h[:, halo:halo + S].double()
    logd = hd @ w.double() + bias
    A = hd.abs() @ w.double().abs() + abs(bias)
    n = 2 * math.ceil(dim / 64) + 6
    delta = _gamma(n, U32) * A
    E = torch.exp(logd)
    v = (E - 1) * factor
    ref = torch.round(v).clamp(1, INT32_MAX)
    eps = factor * (E * (torch.expm1(delta) + 2.0 ** -22) + U32 * (E + 1)) + U32 * v.abs()
    near = (v - torch.floor(v) - 0.5).abs() <= eps
    mask = torch.ones(B, S, dtype=torch.bool, device=dev)
    if lens is not None:
        mask = torch.arange(S, device=dev)[None] < lens_d[:, None]
    ref = torch.where(mask, ref, torch.zeros_like(ref))
    near &= mask & (v < INT32_MAX)
    got = dur.double()
    ok = (got == ref) | (near & ((got - v).abs() <= 0.5 + eps))
    what = f"dim={dim} factor={factor} B={B} S={S} lens={lens} bias={bias}"
    assert ok.all(), f"{what}: {int((~ok).sum())} durations differ, e.g. got {got[~ok][:4].tolist()} want {ref[~ok][:4].tolist()}"
    return int(near.sum())


@gpu
@pytest.mark.parametrize("factor", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("dim", [2, 62, 64, 66, 1280])
def test_durations(dim, factor):
    """B S = 111 (not a multiple of 8 warps per block), NaN halo rows, lens 0 / below S / full and NULL; logd ~ 1 +- 0.8
    gives durations across many .5 boundaries.  Entries within the derived fp32 error of a boundary are counted and
    may round either way; the ASSUMPTIONS #9 audit expects next to none."""
    g = torch.Generator(device=dev).manual_seed(dim * 10 + int(factor * 4))
    near = _dur_case(dim, factor, 3, 37, [37, 0, 20], 1.0, 0.8, g)
    near += _dur_case(dim, factor, 3, 37, None, 1.0, 0.8, g)
    assert near <= 2, f"{near} of 222 durations lie within the fp32 error of a .5 boundary"


@gpu
def test_durations_extremes():
    """logd << 0 gives 1; a duration past 2^31 (logd = 25: 7.2e10; logd = 100: inf in fp32) is clamped to INT32_MAX
    rather than wrapped to its low 32 bits, so that the T2U's max_seq_len check and the vocoder's duration check see it."""
    g = torch.Generator(device=dev).manual_seed(5)
    for bias in (-30.0, -5.0, 25.0, 100.0):
        _dur_case(64, 1.0, 2, 13, [13, 5], bias, 0.05, g)
    lib = _lib()
    h = torch.zeros(1, 64, dtype=torch.float16, device=dev)
    w = torch.zeros(64, dtype=torch.float16, device=dev)
    dur = torch.zeros(1, dtype=torch.int32, device=dev)
    for bias, want in ((25.0, INT32_MAX), (22.0, INT32_MAX), (-30.0, 1)):  # exp(22) - 1 = 3.58e9 > 2^31
        assert lib.sb_durations(h.data_ptr(), 1, 0, w.data_ptr(), bias, 64, None, 1, 1, 1.0, dur.data_ptr(), _stream()) == SB_OK
        assert dur.item() == want, (bias, dur.item())


# ================================================================================================ sb_unit_argmax
def _argmax_case(vocab, U, lens, g, pad=1, eos=2):
    """units = decode(argmax) with the first maximum winning: eos -> pad, pad -> pad + 4, then -4; pad past lens[b].
    Rows hold ties at (i, i + 32), (i, i + 256), (i, i + 2048), all -inf rows, and rows whose argmax is eos or pad; the
    ld - vocab padding columns hold +inf or NaN and the halo rows NaN, none of which may be read."""
    lib = _lib()
    B, halo = len(lens) if lens is not None else 2, 2
    ld = vocab + 7
    rows = U + 2 * halo
    lg = torch.randn(B, rows, ld, device=dev, generator=g)
    lg[:, :, vocab::2] = math.inf
    lg[:, :, vocab + 1::2] = math.nan
    lg[:, :halo] = math.nan
    lg[:, halo + U:] = math.inf
    r = 0
    for gap in (32, 256, 2048):
        for i in (0, 5, vocab // 3):
            if i + gap < vocab and r < B * U:
                lg[r % B, halo + r // B, [i, i + gap]] = 50.0
                r += 1
    if r < B * U:
        lg[r % B, halo + r // B, :vocab] = -math.inf
        r += 1
    for tok in (eos, pad):
        if tok < vocab and r < B * U:
            lg[r % B, halo + r // B, tok] = 60.0
            r += 1
    units = torch.full((B, U), -77, dtype=torch.int32, device=dev)
    lens_d = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    rc = lib.sb_unit_argmax(lg.data_ptr(), ld, rows, halo, U, B, vocab, None if lens_d is None else lens_d.data_ptr(), pad,
                            eos, units.data_ptr(), _stream())
    assert rc == SB_OK, lib.sb_last_error()
    tok = lg[:, halo:halo + U, :vocab].cpu().argmax(-1)  # first maximum
    if lens is not None:
        tok = torch.where(torch.arange(U)[None] < torch.tensor(lens)[:, None], tok, torch.full_like(tok, pad))
    tok = torch.where(tok == eos, torch.full_like(tok, pad), tok)
    tok = torch.where(tok == pad, torch.full_like(tok, pad + 4), tok)
    want = (tok - 4).to(torch.int32)
    assert torch.equal(units.cpu(), want), f"vocab={vocab} U={U} lens={lens}: {int((units.cpu() != want).sum())} differ"


@gpu
@pytest.mark.parametrize("vocab", [1, 7, 256, 257, 10082])
def test_unit_argmax(vocab):
    """Lengths 0, below U and U, and lens = NULL."""
    g = torch.Generator(device=dev).manual_seed(vocab)
    for U in (1, 9, 40):
        _argmax_case(vocab, U, [U, 0, max(1, U // 2)], g)
        _argmax_case(vocab, U, None, g)
