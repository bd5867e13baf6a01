"""Single-token attention of the beam-search step (csrc/decode.cu), called through the C-ABI and checked against a
float64 torch reference built from the same fp16 inputs.

sb_decode_self_attn: one new token per row attends its own ancestry in the KV cache (row r reads position t < step from
cache slot anc[r][t], position `step` is its new k / v) and writes the new k / v to cache[step][r].
sb_decode_cross_attn: the hypotheses of a sentence attend the sentence's encoder K | V (one concatenated buffer, as the
engine passes it), masked to enc_lens.

The sizes straddle every switch inside these entries: the ancestry slots past position 128, the split-K gather's 8/4/1
chunks, the shared-memory cross kernel's staging tail past 32 / 64 frames, its > 48 KB opt-in, its fallback to the
per-row kernel, and the v1 kernels.  Cache positions and encoder frames that no key may read hold NaN, so a stray read
shows in the output.

Bounds.  q / k / v are the fp32 sums bias + partial[0] + partial[1] + ... in that order (the kernels' order) rounded to
fp16, so the new k / v in the cache are compared bit for bit.  The kernels compute in fp32 and round the output to fp16:
|out - ref| <= 2^-11 |ref| (half an fp16 ulp) + 2e-4 max|v| (fp32 sums over up to 3072 keys, __expf)."""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"
HD = 64
SB_OK, SB_ENOSUP = 0, -3  # include/seamless_b200.h


def _lib():
    from seamless_communication_b200 import _lib as L
    return L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _fp32_sum(bias, part):
    """bias + part[0] + part[1] + ... in fp32, left to right (the order of the kernels' gathers), rounded to fp16."""
    acc = bias.clone().expand_as(part[0]).clone()
    for z in range(part.shape[0]):
        acc = acc + part[z]
    return acc.half()


def _check_out(out, ref, vmax, what):
    assert torch.isfinite(out).all(), f"{what}: non-finite output (a NaN-filled cache slot or frame was read)"
    err = (out.double() - ref).abs()
    bound = 2.0 ** -11 * ref.abs() + 2e-4 * vmax
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{what}: error {err.max().item():.3e} is {worst:.2f}x the bound"


# ------------------------------------------------------------------------------------------------ self-attention
def _anc_table(kind, rows, ML, step, g):
    """Ancestor slots anc[r][t] for t < step; the columns from `step` on hold arbitrary valid slots (never to be read)."""
    if kind == "random":
        return torch.randint(0, rows, (rows, ML), generator=g, dtype=torch.int32)
    # a real beam reorder (decode.cu beam_step_kernel): each step, row r continues a parent of its own sentence, inherits
    # the parent's ancestry and reads position `t` from the parent's slot
    beam = 5 if rows % 5 == 0 else rows
    r = torch.arange(rows)
    anc = torch.randint(0, rows, (rows, ML), generator=g)
    for t in range(step):
        parent = (r // beam) * beam + torch.randint(0, beam, (rows,), generator=g)
        anc[:, :t] = anc[parent, :t]
        anc[:, t] = parent
    return anc.to(torch.int32)


def _self_case(ML, step, heads, rows, splits, kind, fp16_qkv=False, seed=0):
    lib = _lib()
    g = torch.Generator().manual_seed(seed * 7919 + ML * 31 + step * 3 + heads + rows * 17 + splits)
    dim = heads * HD
    slice_rows = rows + 3  # partial slices are padded, as ops.slice_rows pads them
    anc = _anc_table(kind, rows, ML, step, g)
    # cache: positions < step hold values only in the slots some row's ancestry names, everything else is NaN
    named = torch.zeros(ML, rows, dtype=torch.bool)
    if step > 0:
        named[torch.arange(step)[None, :].expand(rows, step), anc[:, :step].long()] = True
    kc = torch.full((ML, rows, dim), math.nan, dtype=torch.float16)
    vc = torch.full((ML, rows, dim), math.nan, dtype=torch.float16)
    n = int(named.sum())
    kc[named] = torch.randn(n, dim, generator=g).half()
    vc[named] = torch.randn(n, dim, generator=g).half()
    qscale = torch.ones(3 * dim)
    qscale[:dim] = 2.0  # sharper attention than unit-variance scores
    if fp16_qkv:
        qkv = (torch.randn(rows, 3 * dim, generator=g) * qscale).half()
        part = bias = None
    else:
        part = torch.randn(splits, slice_rows, 3 * dim, generator=g) * qscale / math.sqrt(splits)
        bias = torch.randn(3 * dim, generator=g) * 0.1
        qkv = _fp32_sum(bias, part[:, :rows])
    q, knew, vnew = qkv.view(rows, 3, heads, HD).unbind(1)
    kc_d, vc_d, anc_d = kc.to(dev), vc.to(dev), anc.to(dev)
    out = torch.full((rows, dim), math.nan, dtype=torch.float16, device=dev)
    step_d = torch.tensor([step], dtype=torch.int32, device=dev)
    keep = (part.to(dev), bias.to(dev)) if part is not None else (qkv.to(dev),)
    rc = lib.sb_decode_self_attn(keep[0].data_ptr() if fp16_qkv else None, None if fp16_qkv else keep[0].data_ptr(), splits,
                                 slice_rows, None if fp16_qkv else keep[1].data_ptr(), kc_d.data_ptr(), vc_d.data_ptr(),
                                 anc_d.data_ptr(), ML, step_d.data_ptr(), ML, out.data_ptr(), rows, heads, _stream())
    assert rc == SB_OK, lib.sb_last_error()
    what = f"ML={ML} step={step} heads={heads} rows={rows} splits={splits} anc={kind} fp16_qkv={fp16_qkv}"
    # the new k / v land at [step][r]; nothing else in the caches changes
    kc_new, vc_new = kc.clone(), vc.clone()
    kc_new[step], vc_new[step] = knew.reshape(rows, dim), vnew.reshape(rows, dim)
    assert torch.equal(kc_d.cpu().view(torch.int16), kc_new.view(torch.int16)), f"{what}: K cache"
    assert torch.equal(vc_d.cpu().view(torch.int16), vc_new.view(torch.int16)), f"{what}: V cache"
    # float64 reference over the step + 1 keys of every row
    t_idx = torch.arange(step)[None, :].expand(rows, step)
    K = torch.cat([kc[t_idx, anc[:, :step].long()], knew.reshape(rows, 1, dim)], 1).to(dev, torch.float64).view(rows, step + 1, heads, HD)
    V = torch.cat([vc[t_idx, anc[:, :step].long()], vnew.reshape(rows, 1, dim)], 1).to(dev, torch.float64).view(rows, step + 1, heads, HD)
    s = torch.einsum("rhd,rnhd->rhn", q.to(dev, torch.float64), K) / 8.0
    ref = torch.einsum("rhn,rnhd->rhd", torch.softmax(s, -1), V).reshape(rows, dim)
    _check_out(out, ref, V.abs().max().item(), what)


STEPS = (0, 1, 31, 32, 127, 128, 129, 200)


@pytest.mark.parametrize("kind", ["random", "beam"])
@pytest.mark.parametrize("ML", [102, 263, 1024, 3072])
def test_self_attn_v2_positions(ML, kind):
    """Split-K partials + bias (decode_self_attn2_kernel): every position threshold up to the largest max_len it takes."""
    for step in sorted({s for s in STEPS if s < ML} | {ML - 1}):
        _self_case(ML, step, 5, 7, 5, kind)


@pytest.mark.parametrize("rows", [1, 7, 160])
@pytest.mark.parametrize("heads", [2, 5, 16])
def test_self_attn_v2_shapes(heads, rows):
    for splits in (1, 3, 4, 5, 8, 16):
        for step in (129, 262):
            _self_case(263, step, heads, rows, splits, "random" if splits % 2 else "beam")


@pytest.mark.parametrize("kind", ["random", "beam"])
@pytest.mark.parametrize("ML", [102, 263, 1024, 1536])
def test_self_attn_v1_fp16_qkv(ML, kind):
    """fp16 q | k | v (decode_self_attn_kernel); its scores and slots take 32 B of shared memory per position, so
    max_len <= 1536."""
    for step in sorted({s for s in STEPS if s < ML} | {ML - 1}):
        _self_case(ML, step, 5, 7, 1, kind, fp16_qkv=True)
    for heads, rows in ((2, 1), (16, 160)):
        _self_case(ML, min(200, ML - 1), heads, rows, 1, kind, fp16_qkv=True)


@pytest.mark.parametrize("fp16_qkv,ML", [(False, 3073), (True, 1537)])
def test_self_attn_max_len_too_large_is_refused(fp16_qkv, ML):
    """Past the largest max_len a kernel takes, the entry returns SB_ENOSUP with a message and launches nothing."""
    lib = _lib()
    rows, heads, dim = 2, 2, 128
    kc = torch.zeros(ML, rows, dim, dtype=torch.float16, device=dev)
    vc = torch.zeros_like(kc)
    anc = torch.zeros(rows, ML, dtype=torch.int32, device=dev)
    step = torch.tensor([5], dtype=torch.int32, device=dev)
    qkv = torch.ones(rows, 3 * dim, dtype=torch.float16, device=dev)
    part = torch.ones(1, rows, 3 * dim, device=dev)
    bias = torch.zeros(3 * dim, device=dev)
    out = torch.full((rows, dim), 7.0, dtype=torch.float16, device=dev)
    torch.cuda.synchronize()
    n0 = lib.sb_launch_count()
    rc = lib.sb_decode_self_attn(qkv.data_ptr() if fp16_qkv else None, None if fp16_qkv else part.data_ptr(), 1, rows,
                                 None if fp16_qkv else bias.data_ptr(), kc.data_ptr(), vc.data_ptr(), anc.data_ptr(), ML,
                                 step.data_ptr(), ML, out.data_ptr(), rows, heads, _stream())
    torch.cuda.synchronize()
    assert rc == SB_ENOSUP
    assert b"too large" in lib.sb_last_error()
    assert lib.sb_launch_count() == n0
    assert (out == 7.0).all() and (kc == 0).all() and (vc == 0).all()


# ------------------------------------------------------------------------------------------------ cross-attention
def _cross_case(s_enc, beam, lens_kind, splits=5, fp16_q=False, ragged_rows=False, heads=16, B=3, seed=0):
    lib = _lib()
    g = torch.Generator().manual_seed(seed * 7919 + s_enc * 131 + beam * 7 + splits + 3 * fp16_q + 5 * ragged_rows)
    dim = heads * HD
    rows = B * beam - 1 if ragged_rows else B * beam  # rows % beam != 0: the per-row kernel
    slice_rows = rows + 2
    lens = [s_enc, 1, max(s_enc - 1, 1)][:B] if lens_kind == "ragged" else [s_enc] * B
    kv = torch.randn(B, s_enc, 2 * dim, generator=g).half()
    for b, n in enumerate(lens):
        kv[b, n:] = math.nan  # frames past the valid length are never read
    if fp16_q:
        q = (torch.randn(rows, dim, generator=g) * 2).half()
        part = bias = None
    else:
        part = torch.randn(splits, slice_rows, dim, generator=g) * 2 / math.sqrt(splits)
        bias = torch.randn(dim, generator=g) * 0.1
        q = _fp32_sum(bias, part[:, :rows])
    kv_d = kv.reshape(B * s_enc, 2 * dim).to(dev)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=dev) if lens_kind == "ragged" else None
    out = torch.full((rows, dim), math.nan, dtype=torch.float16, device=dev)
    keep = (q.to(dev),) if fp16_q else (part.to(dev), bias.to(dev))
    rc = lib.sb_decode_cross_attn(keep[0].data_ptr() if fp16_q else None, None if fp16_q else keep[0].data_ptr(), splits,
                                  slice_rows, None if fp16_q else keep[1].data_ptr(), kv_d.data_ptr(), kv_d[:, dim:].data_ptr(),
                                  kv_d.stride(0), None if lens_d is None else lens_d.data_ptr(), s_enc, out.data_ptr(), rows,
                                  beam, heads, _stream())
    assert rc == SB_OK, lib.sb_last_error()
    what = f"s_enc={s_enc} beam={beam} lens={lens_kind} splits={splits} fp16_q={fp16_q} rows%beam={rows % beam}"
    sent = torch.arange(rows, device=dev) // beam
    K = kv_d[:, :dim].view(B, s_enc, heads, HD).double()[sent]
    V = kv_d[:, dim:].view(B, s_enc, heads, HD).double()[sent]
    valid = torch.arange(s_enc, device=dev)[None, :] < torch.tensor(lens, device=dev)[sent][:, None]
    K = torch.where(valid[:, :, None, None], K, 0.0)
    V = torch.where(valid[:, :, None, None], V, 0.0)
    s = torch.einsum("rhd,rnhd->rhn", q.view(rows, heads, HD).to(dev, torch.float64), K) / 8.0
    s = s.masked_fill(~valid[:, None, :], -math.inf)
    ref = torch.einsum("rhn,rnhd->rhd", torch.softmax(s, -1), V).reshape(rows, dim)
    _check_out(out, ref, V.abs().max().item(), what)


S_ENC = (1, 13, 32, 33, 63, 64, 65, 129, 168, 179, 190, 707, 708, 751, 752)
BEAMS = (1, 4, 5, 7)


@pytest.mark.parametrize("lens_kind", ["none", "ragged"])
@pytest.mark.parametrize("beam", BEAMS)
@pytest.mark.parametrize("s_enc", S_ENC)
def test_cross_attn(s_enc, beam, lens_kind):
    """Split-K q partials + bias: the shared-memory kernel (4 warps up to beam 4, 8 above) and, past its shared memory
    limit, the per-row kernel."""
    _cross_case(s_enc, beam, lens_kind)


@pytest.mark.parametrize("s_enc", [13, 65, 190, 752])
def test_cross_attn_v1_entries(s_enc):
    """The per-row kernel (decode_cross_attn_kernel) by fp16 q, and by rows that do not fill whole sentences."""
    for beam in (4, 5, 7):
        for lens_kind in ("none", "ragged"):
            _cross_case(s_enc, beam, lens_kind, fp16_q=True)
            _cross_case(s_enc, beam, lens_kind, ragged_rows=True)


@pytest.mark.parametrize("splits", [1, 3, 4, 5, 8, 16])
def test_cross_attn_splits(splits):
    """The split-K gather's 8-, 4- and 1-slice chunks, on the shared-memory kernel and on the per-row kernel."""
    for s_enc in (65, 190):
        _cross_case(s_enc, 5, "ragged", splits=splits)
        _cross_case(s_enc, 5, "ragged", splits=splits, ragged_rows=True)


def _cross_sweep(order):
    for s_enc in (S_ENC if order == "ascending" else S_ENC[::-1]):
        for beam in BEAMS:
            for lens_kind in ("none", "ragged"):
                _cross_case(s_enc, beam, lens_kind, seed=1)
    torch.cuda.synchronize()


@pytest.mark.parametrize("order", ["ascending", "descending"])
def test_cross_attn_shared_memory_opt_in_in_either_order(order):
    """sb_decode_cross_attn raises the kernel's dynamic shared-memory limit once per process and remembers it: sweep
    s_enc upwards and downwards, each in a fresh process so that no earlier call has configured the limit."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; "
            f"import test_decode_attention as t; t._cross_sweep({order!r}); print('ok')")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout[-2000:] + r.stderr[-4000:]
