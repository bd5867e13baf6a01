"""Thin tensor-level wrappers over the C ABI (include/seamless_b200.h).  PyTorch is used only for device memory and
the current stream; every arithmetic op of the path is one of the CUDA kernels behind these functions."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import BeamDesc, GemmDesc, check

ACT_NONE, ACT_RELU, ACT_SILU, ACT_LRELU, ACT_TANH = 0, 1, 2, 3, 4
F16 = torch.float16


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


class Seq:
    """(B, T, C) fp16 activation in sequence layout: `buf` is (B*Tp, C), data row t of sequence b at b*Tp + PH + t,
    halo rows zero.  lens: optional int32 (B,) valid lengths."""

    __slots__ = ("buf", "B", "T", "C", "PH", "Tp", "lens")

    def __init__(self, B, T, C, halo=0, rows=None, lens=None, dtype=F16, device="cuda", zero=None, buf=None):
        self.B, self.T, self.C, self.PH = B, T, C, halo
        self.Tp = rows if rows is not None else T + 2 * halo
        self.lens = lens
        if buf is not None:
            self.buf = buf
        else:
            zero = (halo > 0 or self.Tp != T) if zero is None else zero
            if zero == "edges":
                # a masked sb_gemm writes every row in [PH, B*Tp-PH) (zeros on halo / padded rows); only the outer
                # PH rows at both ends of the buffer are never touched
                self.buf = torch.empty((B * self.Tp, C), dtype=dtype, device=device)
                if halo > 0:
                    self.buf[:halo].zero_()
                    self.buf[-halo:].zero_()
            else:
                alloc = torch.zeros if zero else torch.empty
                self.buf = alloc((B * self.Tp, C), dtype=dtype, device=device)

    def like(self, C=None, dtype=F16, zero=None):
        return Seq(self.B, self.T, C or self.C, self.PH, self.Tp, self.lens, dtype=dtype, zero=zero)

    def data(self) -> torch.Tensor:
        return self.buf.view(self.B, self.Tp, self.C)[:, self.PH:self.PH + self.T]


def gemm(a: Seq, w: torch.Tensor, n: int, bias=None, *, taps=1, dil=1, act=ACT_NONE, slope=0.0, glu=False, alpha=1.0,
         gamma=1.0, res1: Optional[Seq] = None, res2: Optional[Seq] = None, out: Optional[Seq] = None,
         out2: Optional[Seq] = None, out2_slope=0.0, mask=None, out_f32=False, ref=False, prefetch: Optional[torch.Tensor] = None,
         tile_stats: Optional[torch.Tensor] = None) -> Seq:
    """Linear (taps=1) or 'same'-padded Conv1d (odd taps, dilation dil) over a Seq; output shares a's layout."""
    lib = _lib.load()
    halo = (taps - 1) * dil // 2
    assert halo <= a.PH, f"conv halo {halo} exceeds buffer halo {a.PH}"
    n_out = n // 2 if glu else n
    if out is None:
        out = Seq(a.B, a.T, n_out, a.PH, a.Tp, a.lens, dtype=torch.float32 if out_f32 else F16,
                  zero="edges" if a.PH > 0 else False)
    if mask is None:
        mask = a.PH > 0
    d = GemmDesc()
    d.a, d.a_rows, d.a_ld, d.c_in, d.taps, d.dil = a.buf.data_ptr(), a.B * a.Tp, a.buf.stride(0), a.C, taps, dil
    d.a_row0 = a.PH - halo
    d.w, d.n, d.m = w.data_ptr(), n, a.B * a.Tp - 2 * a.PH
    d.bias, d.act, d.act_slope, d.glu = _p(bias), act, slope, int(glu)
    d.alpha, d.gamma = alpha, gamma
    if res1 is not None:
        d.res1, d.res1_ld = res1.buf.data_ptr(), res1.buf.stride(0)
    if res2 is not None:
        d.res2, d.res2_ld = res2.buf.data_ptr(), res2.buf.stride(0)
    d.out, d.out_ld, d.out_f32 = out.buf.data_ptr(), out.buf.stride(0), int(out_f32)
    if out2 is not None:
        d.out2, d.out2_ld, d.out2_slope = out2.buf.data_ptr(), out2.buf.stride(0), out2_slope
    d.out_row0 = a.PH
    if mask:
        d.seq_rows, d.seq_halo, d.seq_len, d.seq_lens = a.Tp, a.PH, a.T, _p(a.lens)
    if prefetch is not None:
        d.prefetch, d.prefetch_bytes = prefetch.data_ptr(), prefetch.numel() * prefetch.element_size()
    if tile_stats is not None:
        d.tile_stats = tile_stats.data_ptr()
    fn = lib.sb_gemm_ref if ref else lib.sb_gemm
    check(fn(C.byref(d), _stream()), "sb_gemm")
    return out


def gemm_raw(a: torch.Tensor, w: torch.Tensor, n: int, bias=None, *, act=ACT_NONE, glu=False, alpha=1.0, res1=None,
             out=None, out_f32=False, ref=False) -> torch.Tensor:
    """Plain (rows, K) x (n, K)^T on 2-D tensors (row stride = a.stride(0))."""
    lib = _lib.load()
    m, k = a.shape
    n_out = n // 2 if glu else n
    if out is None:
        out = torch.empty((m, n_out), dtype=torch.float32 if out_f32 else F16, device=a.device)
    d = GemmDesc()
    d.a, d.a_rows, d.a_ld, d.c_in, d.taps, d.dil, d.a_row0 = a.data_ptr(), m, a.stride(0), k, 1, 1, 0
    d.w, d.n, d.m = w.data_ptr(), n, m
    d.bias, d.act, d.glu, d.alpha, d.gamma = _p(bias), act, int(glu), alpha, 1.0
    if res1 is not None:
        d.res1, d.res1_ld = res1.data_ptr(), res1.stride(0)
    d.out, d.out_ld, d.out_f32 = out.data_ptr(), out.stride(0), int(out_f32)
    fn = lib.sb_gemm_ref if ref else lib.sb_gemm
    check(fn(C.byref(d), _stream()), "sb_gemm")
    return out


def hifigan_resblock(x: Seq, w1, b1, w2, b2, k: int, dil, *, res2: Optional[Seq] = None, gamma=1.0, out: Seq,
                     out2: Optional[Seq] = None, out2_slope=0.0, slope=0.1) -> Seq:
    """One fused HiFi-GAN ResBlock (hifigan.py:33-121) on a 16- or 32-channel Seq: out = (resblock(x) + res2) * gamma.
    With x.lens, rows past each sequence's length are zero padding and are written as 0."""
    lib = _lib.load()
    assert len(dil) == 3 and len(w1) == len(w2) == len(b1) == len(b2) == 3
    assert x.Tp == x.T + 2 * x.PH and x.buf.stride(0) == x.C
    d = _lib.ResblockDesc()
    d.x, d.res2, d.out, d.out2 = x.buf.data_ptr(), _p(None if res2 is None else res2.buf), out.buf.data_ptr(), _p(
        None if out2 is None else out2.buf)
    for i in range(3):
        d.w1[i], d.b1[i], d.w2[i], d.b2[i] = w1[i].data_ptr(), b1[i].data_ptr(), w2[i].data_ptr(), b2[i].data_ptr()
        d.dilation[i] = dil[i]
    d.channels, d.kernel_size = x.C, k
    d.batch, d.T, d.rows_per_seq, d.halo = x.B, x.T, x.Tp, x.PH
    d.slope, d.gamma, d.out2_slope = slope, gamma, out2_slope
    d.lens = _p(x.lens)
    check(lib.sb_hifigan_resblock(C.byref(d), _stream()), "sb_hifigan_resblock")
    return out


def decode_splits(rows: int, dim: int, ffn_dim: int) -> tuple:
    """K slices (q|k|v, the three dim x dim attention products, FFN out) of the split-K products of a decoder step of
    `rows` rows, on the transposed kernel and on the row-major chain alike.  The slices fix the fp32 summation order
    and with it the search's results, so any change to them is a change of outputs."""
    k_att, k_ffn = max(dim // 64, 1), max(ffn_dim // 64, 1)  # k-blocks of the two residual GEMM kinds
    qkv = max(1, min(2, k_att // 8))
    if rows <= 160 and dim % 64 == 0 and ffn_dim % 64 == 0:
        attn = max(1, min(8, k_att))
    else:
        attn = max(1, min(4, k_att // 4))
    ffn = max(1, min(8, k_ffn // 8))
    while k_att % qkv: qkv -= 1
    while k_att % attn: attn -= 1
    while k_ffn % ffn: ffn -= 1
    return qkv, attn, ffn


def slice_rows(rows: int) -> int:
    """Row stride between split-K slices: padded to the GEMM tile height so the TMA-store epilogue applies."""
    return (rows + 127) // 128 * 128


def gemm_splitk(a: Seq, w: torch.Tensor, n: int, splits: int, partials: torch.Tensor,
                prefetch: Optional[torch.Tensor] = None, transposed=False) -> None:
    """Raw fp32 partial products of a (dense) Seq against w into partials[(z*slice_rows(rows) + r), n]."""
    lib = _lib.load()
    assert a.PH == 0 and a.Tp == a.T
    d = GemmDesc()
    d.a, d.a_rows, d.a_ld, d.c_in, d.taps, d.dil, d.a_row0 = a.buf.data_ptr(), a.B * a.T, a.buf.stride(0), a.C, 1, 1, 0
    d.w, d.n, d.m = w.data_ptr(), n, a.B * a.T
    d.out = partials.data_ptr()  # validated as non-null; sb_gemm_splitk overrides the epilogue fields
    if prefetch is not None:
        d.prefetch, d.prefetch_bytes = prefetch.data_ptr(), prefetch.numel() * prefetch.element_size()
    if transposed and lib.sb_gemm_decode_supported(C.byref(d), splits):
        check(lib.sb_gemm_decode(C.byref(d), splits, partials.data_ptr(), slice_rows(a.B * a.T), _stream()), "sb_gemm_decode")
        return
    check(lib.sb_gemm_splitk(C.byref(d), splits, partials.data_ptr(), slice_rows(a.B * a.T), _stream()), "sb_gemm_splitk")


def gemm_decode(a: Seq, w: torch.Tensor, n: int, bias, act=ACT_NONE, out: Optional[Seq] = None,
                prefetch: Optional[torch.Tensor] = None) -> Seq:
    """out = act(a . w^T + bias) in fp16 for <= 256 rows on the transposed decoder-step kernel (sb_gemm_decode, direct mode)."""
    lib = _lib.load()
    assert a.PH == 0 and a.Tp == a.T
    if out is None:
        out = Seq(a.B, a.T, n)
    d = GemmDesc()
    d.a, d.a_rows, d.a_ld, d.c_in, d.taps, d.dil, d.a_row0 = a.buf.data_ptr(), a.B * a.T, a.buf.stride(0), a.C, 1, 1, 0
    d.w, d.n, d.m = w.data_ptr(), n, a.B * a.T
    d.bias, d.act = _p(bias), act
    d.out, d.out_ld = out.buf.data_ptr(), out.buf.stride(0)
    if prefetch is not None:
        d.prefetch, d.prefetch_bytes = prefetch.data_ptr(), prefetch.numel() * prefetch.element_size()
    check(lib.sb_gemm_decode(C.byref(d), 1, None, 0, _stream()), "sb_gemm_decode")
    return out


def splitk_reduce_ln(partials: torch.Tensor, splits: int, bias, x: Seq, ln_w, ln_b, h: Seq) -> None:
    lib = _lib.load()
    check(lib.sb_splitk_reduce_ln(partials.data_ptr(), splits, x.B * x.T, slice_rows(x.B * x.T), x.C, _p(bias), x.buf.data_ptr(), ln_w.data_ptr(),
                                  ln_b.data_ptr(), h.buf.data_ptr(), _stream()), "sb_splitk_reduce_ln")


def layernorm(x: Seq, w, b, *, res: Optional[Seq] = None, out: Optional[Seq] = None, mask=False) -> Seq:
    lib = _lib.load()
    if out is None:
        out = x.like(zero=x.PH > 0 or x.Tp != x.T)
    assert x.buf.stride(0) == x.C and out.buf.stride(0) == x.C
    check(lib.sb_layernorm(x.buf.data_ptr(), _p(res.buf) if res is not None else None, out.buf.data_ptr(), None,
                           w.data_ptr(), b.data_ptr(), x.C, x.B, x.T, x.Tp, x.PH, out.Tp, out.PH, _p(x.lens),
                           int(mask and x.lens is not None), _stream()), "sb_layernorm")
    return out


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, B, H, sq, sk, q_rows, q_halo,
              kv_rows, kv_halo, kv_lens=None, causal=False, rel_k=None, rel_left=0, rel_right=0):
    """q/k/v/out are 2-D views whose row 0 is row 0 of sequence 0 (column offsets select q|k|v inside fused buffers)."""
    lib = _lib.load()
    check(lib.sb_attention(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                           out.data_ptr(), out.stride(0), B, H, sq, sk, q_rows, q_halo, kv_rows, kv_halo, _p(kv_lens),
                           int(causal), _p(rel_k), rel_left, rel_right, _stream()), "sb_attention")
    return out


def self_attention(qkv: Seq, H: int, *, causal=False, rel_k=None, rel_left=0, rel_right=0) -> Seq:
    M = qkv.C // 3
    out = Seq(qkv.B, qkv.T, M, qkv.PH, qkv.Tp, qkv.lens, zero=qkv.PH > 0)
    b = qkv.buf
    attention(b[:, 0:M], b[:, M:2 * M], b[:, 2 * M:3 * M], out.buf, qkv.B, H, qkv.T, qkv.T, qkv.Tp, qkv.PH, qkv.Tp,
              qkv.PH, qkv.lens, causal, rel_k, rel_left, rel_right)
    return out


def attention_relpos(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, B, H, S, q_rows, q_halo, kv_rows,
                     kv_halo, r: torch.Tensor, u=None, vb=None, kv_lens=None):
    """Transformer-XL relative attention (sb_attention_relpos); r is (2S-1, H*64) fp16, u / vb fp32 (H, 64) or None."""
    lib = _lib.load()
    check(lib.sb_attention_relpos(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                  out.data_ptr(), out.stride(0), B, H, S, q_rows, q_halo, kv_rows, kv_halo, _p(kv_lens),
                                  r.data_ptr(), r.stride(0), _p(u), _p(vb), _stream()), "sb_attention_relpos")
    return out


def self_attention_relpos(qkv: Seq, H: int, r: torch.Tensor, u=None, vb=None) -> Seq:
    M = qkv.C // 3
    out = Seq(qkv.B, qkv.T, M, qkv.PH, qkv.Tp, qkv.lens, zero=qkv.PH > 0)
    b = qkv.buf
    attention_relpos(b[:, 0:M], b[:, M:2 * M], b[:, 2 * M:3 * M], out.buf, qkv.B, H, qkv.T, qkv.Tp, qkv.PH, qkv.Tp, qkv.PH, r,
                     u, vb, qkv.lens)
    return out


def dwconv_bias_silu(x: Seq, w, bias, k: int) -> Seq:
    """w2v-BERT v1 depthwise conv (symmetric padding) + per-channel bias (BatchNorm folded into w) + SiLU."""
    lib = _lib.load()
    assert x.PH == 0 and x.Tp == x.T
    y = x.like()
    check(lib.sb_dwconv_bias_silu(x.buf.data_ptr(), y.buf.data_ptr(), w.data_ptr(), bias.data_ptr(), x.B, x.T, x.C, k,
                                  _stream()), "sb_dwconv_bias_silu")
    return y


def dwconv_ln_silu(x: Seq, w, ln_w, ln_b, k: int) -> Seq:
    lib = _lib.load()
    assert x.PH == 0 and x.Tp == x.T
    y = x.like()
    check(lib.sb_dwconv_ln_silu(x.buf.data_ptr(), y.buf.data_ptr(), w.data_ptr(), ln_w.data_ptr(), ln_b.data_ptr(),
                                x.B, x.T, x.C, k, _stream()), "sb_dwconv_ln_silu")
    return y


def fbank(wave: torch.Tensor, num_samples: torch.Tensor, frames_ld: int, standardize=True):
    """wave (B, Tmax) fp32 cuda, num_samples (B,) int32 cuda -> (B, frames_ld, 80) fp16, frames (B,) int32"""
    lib = _lib.load()
    B = wave.shape[0]
    out = torch.empty((B, frames_ld, 80), dtype=F16, device=wave.device)
    work = torch.empty((B, frames_ld, 80), dtype=torch.float32, device=wave.device)
    frames = torch.empty((B,), dtype=torch.int32, device=wave.device)
    check(lib.sb_fbank(wave.data_ptr(), wave.stride(0), num_samples.data_ptr(), B, out.data_ptr(), frames_ld,
                       work.data_ptr(), frames.data_ptr(), int(standardize), _stream()), "sb_fbank")
    return out, frames


def embed_seq(ids: torch.Tensor, embed, pos, scale, dim) -> torch.Tensor:
    lib = _lib.load()
    R, L = ids.shape
    x = torch.empty((R * L, dim), dtype=F16, device=ids.device)
    check(lib.sb_embed_seq(ids.data_ptr(), ids.stride(0), L, embed.data_ptr(), pos.data_ptr(), scale, x.data_ptr(), R,
                           dim, _stream()), "sb_embed_seq")
    return x


def launch_count() -> int:
    return int(_lib.load().sb_launch_count())
