"""decode_gemm.cu (sb_gemm_decode, the transposed wgmma kernel behind all six weight products of a beam-search step)
against float64 at every decoder-step shape of seamlessM4T_large, at the row counts the searches run (160 = 32 x beam 5,
40 = the s2tt batch of 8 x 5, and ragged ones), at the splits a step uses, one split and an uneven split; bit for bit
against the row-major kernels at the step's splits; and one whole search on the default (transposed) path against the
row-major launch chain."""
import math

import pytest
import torch

from seamless_communication_b200.ops import decode_splits

pytestmark = pytest.mark.gpu
dev = "cuda"
ROWS = [160, 5, 37, 40, 256]
M, FFN = 1024, 8192


@pytest.fixture(scope="module")
def ops():
    from seamless_communication_b200 import ops as _ops
    return _ops


def _operands(rows, n, k, seed):
    from seamless_communication_b200.ops import Seq
    g = torch.Generator(device=dev).manual_seed(seed)
    a = Seq(1, rows, k, buf=torch.randn(rows, k, device=dev, generator=g).half())
    w = (torch.randn(n, k, device=dev, generator=g) / math.sqrt(k)).half()
    bias = torch.randn(n, device=dev, generator=g)
    ref = a.buf.double() @ w.double().t()
    return a, w, bias, ref


def step_splits(rows):
    """K splits of a seamlessM4T_large step of `rows` rows (engine._search_state), per (n, k) product"""
    qkv, attn, ffn = decode_splits(rows, M, FFN)
    return {(3 * M, M): qkv, (M, M): attn, (M, FFN): ffn}


STEP_SPLITS = step_splits(160)  # the bench step's splits, which the float64 tests try at every row count


def _split_choices(n, k):
    """the step's split count, one split, and an uneven one (slices of different k-block counts)"""
    kb = k // 64
    uneven = next(s for s in range(min(kb, 5), 0, -1) if kb % s or s == 1)
    return sorted({STEP_SPLITS[(n, k)], 1, uneven})


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("n,k", [(3 * M, M), (M, M), (M, FFN)], ids=["qkv", "attn", "ffn_out"])
def test_splitk_matches_float64(ops, rows, n, k):
    """split-K partials (q|k|v, the three 1024 x 1024 attention products, FFN out): every slice this call writes sums to
    the float64 product; rows past `rows` and slices past `splits` keep their NaN; a repeated call is bit-identical."""
    a, w, _, ref = _operands(rows, n, k, rows * 7 + n + k)
    SR = ops.slice_rows(rows)
    for splits in _split_choices(n, k):
        part = torch.full(((splits + 1) * SR, n), float("nan"), device=dev)
        ops.gemm_splitk(a, w, n, splits, part, transposed=True)
        p = part.view(splits + 1, SR, n)
        assert not torch.isnan(p[:splits, :rows]).any(), splits
        assert torch.isnan(p[:splits, rows:]).all() and torch.isnan(p[splits]).all(), splits
        err = (p[:splits, :rows].double().sum(0) - ref).abs().max().item()
        assert err < 1e-3, (splits, err)
        again = torch.full_like(part, float("nan"))
        ops.gemm_splitk(a, w, n, splits, again, transposed=True)
        assert torch.equal(p[:splits, :rows], again.view(splits + 1, SR, n)[:splits, :rows]), splits


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("n,k", [(FFN, M), (1126, 128), (FFN, 64)], ids=["ffn_inner", "ragged", "one_kblock"])
def test_direct_bias_relu_matches_float64(ops, rows, n, k):
    """direct mode (FFN inner: fp16 out = relu(a . w^T + bias)), plus a ragged last feature tile (n % 8 != 0: the scalar
    store path) and a single k-block.  Columns past n and rows past `rows` of a wider output keep their NaN; a repeated
    call is bit-identical."""
    from seamless_communication_b200.ops import Seq
    a, w, bias, ref = _operands(rows, n, k, rows * 11 + n + k)
    want = torch.relu(ref + bias.double())
    big = torch.full((rows + 3, n + 8), float("nan"), device=dev).half()
    out = Seq(1, rows, n, buf=big[:rows, :n])
    ops.gemm_decode(a, w, n, bias, act=ops.ACT_RELU, out=out)
    got = big[:rows, :n].double()
    assert ((got - want).abs() <= 2e-3 + 1e-3 * want.abs()).all(), (got - want).abs().max().item()
    assert torch.isnan(big[rows:]).all() and torch.isnan(big[:, n:]).all()
    first = big.clone()
    ops.gemm_decode(a, w, n, bias, act=ops.ACT_RELU, out=out)
    assert torch.equal(big[:rows, :n], first[:rows, :n])
    lin = ops.gemm_decode(a, w, n, None)  # no bias, no activation
    assert ((lin.buf.double() - ref).abs() <= 2e-3 + 1e-3 * ref.abs()).all()


@pytest.mark.parametrize("rows", ROWS)
def test_bit_identical_to_row_major_kernels_at_step_slices(ops, rows):
    """At the step's K slices the transposed kernel sums the same k-blocks in the same order as the kernels of the
    row-major chain (sb_gemm_splitk, sb_gemm for FFN inner), so its partials and its fp16 FFN output are bit-identical
    to theirs and a search does not depend on the path."""
    from seamless_communication_b200.ops import Seq
    SR = ops.slice_rows(rows)
    for (n, k), splits in step_splits(rows).items():
        a, w, _, _ = _operands(rows, n, k, rows * 13 + n + k)
        want, got = (torch.zeros(splits * SR, n, device=dev) for _ in range(2))
        ops.gemm_splitk(a, w, n, splits, want)
        ops.gemm_splitk(a, w, n, splits, got, transposed=True)
        assert torch.equal(got.view(splits, SR, n)[:, :rows], want.view(splits, SR, n)[:, :rows]), (n, k, splits)
    a, w, bias, _ = _operands(rows, FFN, M, rows * 17)
    want = ops.gemm(a, w, FFN, bias, act=ops.ACT_RELU, out=Seq(1, rows, FFN))
    got = ops.gemm_decode(a, w, FFN, bias, act=ops.ACT_RELU, out=Seq(1, rows, FFN))
    assert torch.equal(got.buf, want.buf)


def test_search_step_transposed_equals_launch_chain():
    """A beam search of 32 sentences x beam 5 (160 rows, the bench's step) on `small`: the default path (all six products
    on sb_gemm_decode) against decode_gemm_t = False (the row-major chain), at the same K slices: the hypotheses,
    their scores and the final-LayerNorm state of every step are identical; and a second default search is too."""
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.ops import Seq
    eng = load_unity_model("small_v2", synthetic=True, seed=7, dec_gain=4.0).engine
    cfg = eng.cfg
    torch.manual_seed(23)
    M_, S_enc, B, beam = cfg.model_dim, 13, 32, 5
    e = Seq(B, S_enc, M_, buf=torch.randn(B * S_enc, M_, device=dev).half())
    lens = torch.randint(3, S_enc + 1, (B,), dtype=torch.int32, device=dev)
    lens[0] = S_enc
    prefix = [cfg.text_eos, eng.text_tokenizer.lang_index("spa")]
    assert eng.decode_gemm_t and not eng.decode_fused
    runs = {}
    try:
        for gemm_t in (True, False, True):
            eng.decode_gemm_t = gemm_t
            hyps = eng.beam_search(e, lens, prefix, beam=beam, soft_max=(1, 9), hard_max=40)
            st = eng._last_search_states[0]
            assert st["gemm_t"] == gemm_t and st["R"] == 160
            n = min(len(h[0][1]) for h in hyps) - 1
            run = (hyps, st["hist"][:n].clone())
            if gemm_t and gemm_t in runs:  # determinism: the second default search is bit-identical
                assert [h[0][1] for h in hyps] == [h[0][1] for h in runs[True][0]]
                assert torch.equal(run[1], runs[True][1][:run[1].shape[0]])
            runs.setdefault(gemm_t, run)
    finally:
        eng.decode_gemm_t = True
    (h_t, hist_t), (h_c, hist_c) = runs[True], runs[False]
    assert [[x[1] for x in h] for h in h_t] == [[x[1] for x in h] for h in h_c]
    assert [[x[0] for x in h] for h in h_t] == [[x[0] for x in h] for h in h_c]
    assert torch.equal(hist_t, hist_c)
