"""UnitY2 forced aligner (DESIGN.md section 12): the oracle, config, state-dict names, converter and tokenisation against
the reference's own code (tests/golden/aligner.npz) and the API's argument checks on the CPU; both kernels against
float64, the engine against the oracle, ragged batches and the audio -> units -> alignment path on the GPU."""
import math
import os
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle_aligner as O  # noqa: E402
from seamless_communication_b200 import config as C  # noqa: E402
from seamless_communication_b200 import synthetic as S  # noqa: E402
from seamless_communication_b200.models.checkpoint import convert_unity2_aligner_checkpoint  # noqa: E402

FX = np.load(os.path.join(ROOT, "tests", "golden", "aligner.npz"))
U32 = 2.0 ** -24  # fp32 unit roundoff
U16 = 2.0 ** -11  # fp16 unit roundoff


# ------------------------------------------------------------------------------------------------------------ CPU
def test_config_fields_equal_the_reference_architecture():
    cfg = C.nar_t2u_aligner()
    for k in ("model_dim", "feat_dim", "num_text_layers", "num_feat_layers", "dropout", "temperature", "reduction_factor"):
        assert getattr(cfg, k) == FX[f"arch.{k}"].item(), k
    assert (cfg.unit_vocab_size, cfg.unit_unk_idx, cfg.unit_bos_idx, cfg.unit_eos_idx, cfg.unit_pad_idx) == tuple(
        FX[f"arch.unit_vocab.{k}"].item() for k in ("size", "unk_idx", "bos_idx", "eos_idx", "pad_idx"))
    assert cfg.text_vocab_size == FX["arch.text_vocab_size"].item()
    assert cfg.name == FX["arch.model_name_or_card"].item() == FX["card.model_arch"].item()
    assert cfg.num_units == FX["card.num_units"].item()
    assert list(cfg.unit_langs) == FX["card.unit_langs"].tolist()
    tiny = C.tiny_aligner()
    assert (tiny.num_text_layers, tiny.num_feat_layers, tiny.reduction_factor) == (2, 3, 1)
    assert tiny.unit_vocab_size == tiny.num_units + 2 * (len(tiny.unit_langs) + 1) + 4


def test_state_dict_names_and_shapes_equal_the_reference():
    for cfg in (C.tiny_aligner(),):
        sd = S.make_aligner_state_dict(cfg)
        enc = {k[len("alignment_encoder."):]: tuple(v.shape) for k, v in sd.items() if k.startswith("alignment_encoder.")}
        assert list(enc) == FX["encoder.keys"].tolist()
        W = 16  # the fixture's width
        for k, shp in zip(FX["encoder.keys"].tolist(), FX["encoder.shapes"].tolist()):
            ref = tuple(cfg.model_dim if int(d) == W else int(d) for d in shp.split(","))
            assert enc[k] == ref, (k, enc[k], ref)
        assert tuple(sd["alignment_frontend.embed_text.weight"].shape) == (cfg.text_vocab_size, cfg.model_dim)
        assert tuple(sd["alignment_frontend.embed_unit.weight"].shape) == (cfg.unit_vocab_size, cfg.feat_dim)


def _golden_generator():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_aligner", os.path.join(ROOT, "tests", "golden", "make_golden_aligner.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_oracle_encoder_equals_the_reference():
    """lprob within float64 rounding (1e-12 relative to the scores), durations exactly, in both row-0 orders."""
    gen = _golden_generator()
    for seed, T_text, T_feat in gen.ENCODER_CASES:
        sd = gen.encoder_state_dict(seed)
        t, f = gen.encoder_inputs(seed, T_text, T_feat)
        lp, tt, ff = O.encoder_lprob(sd, t[0], f[0])
        ref = torch.from_numpy(FX[f"encoder.{seed}.lprob"])
        assert lp.shape == ref.shape == (T_feat, T_text)
        scale = max(1.0, ref.abs().max().item())
        assert (lp - ref).abs().max().item() <= 1e-12 * scale, seed
        dur = FX[f"encoder.{seed}.durations"]
        for numpy_row0 in (False, True):
            got = O.durations(lp.float().numpy(), numpy_row0)
            assert got.tolist() == dur.tolist() + [0] * (T_text - len(dur)), (seed, numpy_row0)


@pytest.mark.parametrize("case", ["ties", "neg_inf", "planted", "short", "one_text", "one_feat", "random"])
def test_oracle_search_equals_the_reference(case):
    lp = FX[f"mas.{case}.lprob"]
    for numpy_row0 in (False, True):
        assert O.mas_path(lp, numpy_row0).tolist() == FX[f"mas.{case}.path"].tolist(), numpy_row0
    if case == "planted":
        assert FX["mas.planted.durations"].tolist() == [3, 1, 5, 2, 4]


def test_converter_equals_the_reference():
    pieces = FX["convert.pieces"].tolist()
    ck = {src: {} for src in ("text_emb_state", "unit_emb_state", "aligner_state")}
    for k in FX.files:
        if k.startswith("convert.in."):
            src, name = k[len("convert.in."):].split(".", 1)
            ck[src][name] = torch.from_numpy(FX[k].copy())
    before = ck["text_emb_state"]["weight"].clone()
    out = convert_unity2_aligner_checkpoint(ck, pieces)["model"]
    assert sorted(out) == sorted(FX["convert.keys"].tolist())
    for k, v in out.items():
        assert torch.equal(v, torch.from_numpy(FX[f"convert.out.{k}"])), k
    assert torch.equal(ck["text_emb_state"]["weight"], before)  # the caller's table is not permuted in place
    assert convert_unity2_aligner_checkpoint({"model": out}, pieces)["model"] is out


def test_unit_tokenisation_equals_the_reference():
    from seamless_communication_b200.models.aligner import UnitY2AlignmentFrontend
    fe = UnitY2AlignmentFrontend(C.nar_t2u_aligner(), S.SyntheticCharTokenizer(64))
    assert fe.unit_tokenizer.vocab_info.size == FX["units.vocab_size"].item()
    assert fe.tokenize_unit(torch.from_numpy(FX["units.in"])).tolist() == FX["units.out"].tolist()
    assert fe.tokenize_unit("7 10003 10004 0").tolist() == FX["units.out_str"].tolist()


def test_char_tokenisation_equals_sentencepiece(tmp_path):
    spm = pytest.importorskip("sentencepiece")
    corpus = tmp_path / "c.txt"
    corpus.write_text("the quick brown fox jumps over the lazy dog\nécole café naïve Ärger\nＡＢＣ full width\n" * 20)
    spm.SentencePieceTrainer.train(input=str(corpus), model_prefix=str(tmp_path / "ch"), model_type="char", vocab_size=45,
                                   character_coverage=1.0, minloglevel=2)
    sp = spm.SentencePieceProcessor(model_file=str(tmp_path / "ch.model"))
    texts = ["the fox", "  the   fox  ", "\tthe\tfox\t", "école", "école", "ÄRGER café", "ＡＢＣ ｄｏｇ", "x!q #",
             "", "   ", "a　b", "a\nb\r\nc", "the examination and testimony of the experts"]
    known = lambda p: sp.piece_to_id(p) != sp.unk_id()  # noqa: E731
    for t in texts:
        assert [sp.piece_to_id(p) for p in S.char_pieces(t, known)] == sp.encode(t), repr(t)
        assert S.char_pieces(t, known) == sp.encode(t, out_type=str), repr(t)
    assert sp.encode("x!q #")[-1] == sp.unk_id()  # characters the model lacks
    assert len(sp.encode("ÄRGER")) == 3  # a run of them is one unknown piece
    # the product's frontend encodes through the same function, given only the tokenizer's piece model
    from types import SimpleNamespace
    from seamless_communication_b200.models.aligner import UnitY2AlignmentFrontend
    tok = SimpleNamespace(model=SimpleNamespace(token_to_index=sp.piece_to_id, index_to_token=sp.id_to_piece),
                          vocab_info=S.VocabularyInfo(sp.get_piece_size(), sp.unk_id(), sp.bos_id(), sp.eos_id(), sp.pad_id()))
    fe = UnitY2AlignmentFrontend(C.tiny_aligner(), tok)
    for t in texts:
        assert fe.tokenize_text(t).tolist() == sp.encode(t), repr(t)
        assert fe.tokenize_text_to_tokens(t) == sp.encode(t, out_type=str), repr(t)


def test_reference_sentence_gives_115_ids():
    from seamless_communication_b200.models.aligner import UnitY2AlignmentFrontend
    fe = UnitY2AlignmentFrontend(C.tiny_aligner(), S.SyntheticCharTokenizer(64))
    text = ("the examination and testimony of the experts enabled the commision to conclude that five shots may have "
            "been fired")
    assert len(text) == 114
    ids = fe.tokenize_text(text)
    assert len(ids) == 115 and len(fe.tokenize_text(text, add_trailing_silence=True)) == 116
    assert fe.tokenize_text(text, add_trailing_silence=True)[-1] == ids[0]
    assert fe.decode_text(ids) == text


def _cpu_extractor():
    """An AlignmentExtractor whose tokenisation and argument checks run without a GPU (no engine is built)."""
    from seamless_communication_b200.models.aligner import AlignmentExtractor, UnitY2AlignmentFrontend, UnitY2AlignmentModel
    cfg = C.tiny_aligner()
    ex = AlignmentExtractor.__new__(AlignmentExtractor)
    ex.device, ex.dtype, ex.unit_extractor, ex.unit_extractor_output_layer = torch.device("cpu"), torch.float16, None, 0
    ex.alignment_model = UnitY2AlignmentModel(cfg, UnitY2AlignmentFrontend(cfg, S.SyntheticCharTokenizer(64)), None)
    return ex


def test_api_errors():
    from seamless_communication_b200.aligner_engine import AlignerEngine
    from seamless_communication_b200.models.aligner import AlignmentExtractor, load_unity2_alignment_model
    with pytest.raises(RuntimeError, match="no weights"):
        load_unity2_alignment_model("tiny_aligner", char_tokenizer=S.SyntheticCharTokenizer(64))
    with pytest.raises(RuntimeError, match="character tokenizer"):
        load_unity2_alignment_model("tiny_aligner", state_dict={})
    with pytest.raises(ValueError, match="unknown"):
        load_unity2_alignment_model("aligner_nonexistent", synthetic=True)
    with pytest.raises(ValueError, match="URL"):
        AlignmentExtractor("tiny_aligner", "tiny_xlsr", 3, "https://example.org/kmeans_10k.npy", synthetic=True)
    with pytest.raises(ValueError, match="reduction_factor"):
        AlignerEngine(replace(C.tiny_aligner(), reduction_factor=2), {})
    ex = _cpu_extractor()
    units = torch.tensor([5, 6, 7])
    with pytest.raises(NotImplementedError, match="matplotlib"):
        ex.extract_alignment(units, "abc", plot=True)
    with pytest.raises(ValueError, match="empty text"):
        ex.extract_alignment(units, "   ")
    with pytest.raises(ValueError, match="no units"):
        ex.extract_alignment(torch.zeros(0, dtype=torch.int64), "abc")
    with pytest.raises(ValueError, match="Channel > Time"):
        ex.prepare_audio(torch.zeros(5, 3))
    with pytest.raises(ValueError, match="unit extractor"):
        ex.extract_alignment(torch.zeros(16000), "abc")
    assert torch.equal(ex.prepare_audio(torch.tensor([[1.0, 2.0, 3.0], [3.0, 4.0, 5.0]])), torch.tensor([2.0, 3.0, 4.0]))


def test_prepare_audio_averages_wav_channels_and_refuses_other_rates(tmp_path):
    import struct
    ex = _cpu_extractor()
    x = np.stack([np.linspace(-0.5, 0.5, 800), np.linspace(0.25, -0.25, 800)], 1).astype("<f4")

    def write(path, rate):
        body = x.tobytes()
        fmt = struct.pack("<HHIIHH", 3, 2, rate, rate * 8, 8, 32)
        with open(path, "wb") as f:
            f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt) + 8 + len(body)) + b"WAVE")
            f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(body)) + body)

    write(tmp_path / "a.wav", 16000)
    got = ex.prepare_audio(str(tmp_path / "a.wav"))
    assert torch.allclose(got, torch.from_numpy(x.mean(1)), atol=1e-7)
    from seamless_communication_b200.evaluate import decode_wav
    assert torch.equal(decode_wav(str(tmp_path / "a.wav")), torch.from_numpy(x[:, 0].copy()))  # default: channel 0
    write(tmp_path / "b.wav", 22050)
    with pytest.raises(ValueError, match="22050"):
        ex.prepare_audio(str(tmp_path / "b.wav"))


# ------------------------------------------------------------------------------------------------------------ GPU
def _lib():
    from seamless_communication_b200 import _lib as L
    return L.load()


def _run_lprob(f_rows, t_rows, feat_lens, text_lens, dim, T_feat, T_text, temperature=1.0, pad=3):
    """f_rows (B, T_feat + 2, dim) / t_rows (B, T_text + 2, dim) fp32 with one halo row on each side; output with
    `pad` sentinel columns after T_text."""
    from seamless_communication_b200 import ops
    B = len(feat_lens)
    out = torch.full((B, T_feat, T_text + pad), 7.0, device="cuda")
    f, t = f_rows.reshape(-1, dim).cuda(), t_rows.reshape(-1, dim).cuda()
    fl, tl = torch.tensor(feat_lens, dtype=torch.int32).cuda(), torch.tensor(text_lens, dtype=torch.int32).cuda()
    rc = _lib().sb_align_lprob(f.data_ptr(), dim, T_feat + 2, 1, fl.data_ptr(), t.data_ptr(), dim, T_text + 2, 1, tl.data_ptr(),
                               dim, B, T_feat, T_text, temperature, out.data_ptr(), T_text + pad, ops._stream())
    assert rc == 0
    return out.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("dim,T_text,feat_lens,text_lens", [
    (64, 1, [1, 63, 64, 65], [1, 1, 1, 1]),
    (64, 2, [2001, 5], [2, 1]),
    (64, 31, [130, 64], [31, 17]),
    (80, 32, [100, 1], [32, 32]),
    (64, 33, [65, 129], [33, 1]),
    (1024, 1100, [300, 70], [1100, 513]),
])
def test_align_lprob_against_float64(dim, T_text, feat_lens, text_lens):
    """Bound per frame j, from fp32 arithmetic on exact fp32 inputs: each (f - t)^2 term carries <= 3u relative error
    (difference, square, add) and the in-order sum of dim non-negative terms <= dim*u of the total, so d^2 is within
    (dim + 3) u relative and d = sqrt(d^2) within ((dim + 3)/2 + 1) u; the scores' error E_j <= temperature *
    ((dim + 5)/2) u * max_i d_i.  The log-sum-exp moves by at most E_j, plus the fp32 exp / log / sum roundings, bounded by
    4 u (|lse| + max|s|) + 4 N u.  So |lp - lp64| <= 2 E_j + 4 u (|lse| + max|s|) + 4 N u.
    Inputs past a row's length and in the halo rows hold NaN (never read); sentinel columns past T_text, and the
    columns of tokens past text_len (-inf) and frames past feat_len (0), are checked exactly."""
    T_feat = max(feat_lens)
    B = len(feat_lens)
    g = torch.Generator().manual_seed(dim + T_text)
    f = torch.full((B, T_feat + 2, dim), float("nan"))
    t = torch.full((B, T_text + 2, dim), float("nan"))
    for b in range(B):
        f[b, 1:1 + feat_lens[b]] = torch.randn(feat_lens[b], dim, generator=g)
        t[b, 1:1 + text_lens[b]] = torch.randn(text_lens[b], dim, generator=g) + 0.3
    temperature = 0.7
    out = _run_lprob(f, t, feat_lens, text_lens, dim, T_feat, T_text, temperature)
    assert (out[:, :, T_text:] == 7.0).all()
    for b in range(B):
        F_, N = feat_lens[b], text_lens[b]
        ff, tt = f[b, 1:1 + F_].double(), t[b, 1:1 + N].double()
        d = torch.cat([(ff[j:j + 64, None] - tt[None]).pow(2).sum(-1).sqrt() for j in range(0, F_, 64)])
        s = -temperature * d
        ref = torch.log_softmax(s, -1)
        lse = torch.logsumexp(s, -1, keepdim=True)
        E = temperature * (dim + 5) / 2 * U32 * d.max(-1, keepdim=True).values
        bound = 2 * E + 4 * U32 * (lse.abs() + s.abs().max(-1, keepdim=True).values) + 4 * N * U32
        err = (out[b, :F_, :N].double() - ref).abs()
        assert (err <= bound).all(), (b, (err - bound).max().item())
        assert (out[b, :F_, N:T_text] == float("-inf")).all()
        assert (out[b, F_:, :T_text] == 0).all()


def _mas_gpu(lp_rows, feat_lens, text_lens, T_feat, T_text):
    from seamless_communication_b200 import ops
    lp = lp_rows.cuda()
    dur, path = ops.monotonic_align(lp, torch.tensor(feat_lens, dtype=torch.int32).cuda(),
                                    torch.tensor(text_lens, dtype=torch.int32).cuda(), path=True)
    return dur.cpu(), path.cpu()


def _random_lprob(F_, N, g, sharp=3.0):
    return torch.log_softmax(sharp * torch.randn(F_, N, generator=g), -1)


@pytest.mark.gpu
def test_monotonic_align_bit_exact_against_float64():
    """Paths and durations equal the float64 restatement (oracle_aligner.mas_q: same order, same float64 arithmetic)
    exactly, on random lprob with ragged lengths; padding holds NaN (never read); edge cases T_feat < T_text, T_text = 1,
    T_feat = 1, and rows longer than the 8 rows per lane loaded a column ahead."""
    shapes = [(500, 150), (1, 1), (1, 7), (7, 1), (3, 9), (2000, 300), (64, 64), (33, 32), (900, 1100), (40, 256), (257, 33)]
    feat_lens, text_lens = [s[0] for s in shapes], [s[1] for s in shapes]
    T_feat, T_text = max(feat_lens), max(text_lens)
    g = torch.Generator().manual_seed(11)
    lp = torch.full((len(shapes), T_feat, T_text), float("nan"))
    for b, (F_, N) in enumerate(shapes):
        lp[b, :F_, :N] = _random_lprob(F_, N, g)
    dur, path = _mas_gpu(lp, feat_lens, text_lens, T_feat, T_text)
    for b, (F_, N) in enumerate(shapes):
        A = O.mas_path(lp[b, :F_, :N].numpy())
        assert path[b, :F_].tolist() == A.tolist(), (F_, N)
        assert (path[b, F_:] == -1).all()
        assert dur[b, :N].tolist() == np.bincount(A, minlength=N).tolist(), (F_, N)
        assert (dur[b, N:] == 0).all() and int(dur[b].sum()) == F_


@pytest.mark.gpu
def test_monotonic_align_equals_the_reference_fixture():
    """The fixture's crafted matrices (exact ties, -inf entries, planted blocks, T_feat < T_text, T_text = 1,
    T_feat = 1) and the encoder cases, one row each in one ragged batch."""
    mats = [FX[f"mas.{c}.lprob"] for c in ("ties", "neg_inf", "planted", "short", "one_text", "one_feat", "random")]
    want = [FX[f"mas.{c}.path"] for c in ("ties", "neg_inf", "planted", "short", "one_text", "one_feat", "random")]
    gen = _golden_generator()
    for seed, _, _ in gen.ENCODER_CASES:
        mats.append(FX[f"encoder.{seed}.lprob"].astype(np.float32))
        want.append(None)
    fl, tl = [m.shape[0] for m in mats], [m.shape[1] for m in mats]
    lp = torch.full((len(mats), max(fl), max(tl)), float("nan"))
    for b, m in enumerate(mats):
        lp[b, :fl[b], :tl[b]] = torch.from_numpy(m)
    dur, path = _mas_gpu(lp, fl, tl, max(fl), max(tl))
    for b, m in enumerate(mats):
        if want[b] is not None:
            assert path[b, :fl[b]].tolist() == want[b].tolist(), b
        else:
            seed = gen.ENCODER_CASES[b - 7][0]
            ref = FX[f"encoder.{seed}.durations"].tolist()
            assert dur[b, :tl[b]].tolist() == ref + [0] * (tl[b] - len(ref)), seed
    assert dur[2, :5].tolist() == [3, 1, 5, 2, 4]
    assert dur[0, :3].tolist() == FX["mas.ties.durations"].tolist()  # ties go to the lower index


@pytest.mark.gpu
def test_monotonic_align_recovers_planted_durations_and_refuses_long_texts():
    g = torch.Generator().manual_seed(5)
    rows = []
    for n in (1, 5, 40, 300):
        d = torch.randint(1, 6, (n,), generator=g)
        lp = torch.log(torch.full((int(d.sum()), n), 0.02))
        j = 0
        for i, k in enumerate(d.tolist()):
            lp[j:j + k, i] = math.log(0.9)
            j += k
        rows.append((d, lp))
    fl, tl = [r[1].shape[0] for r in rows], [r[1].shape[1] for r in rows]
    lp = torch.full((len(rows), max(fl), max(tl)), float("nan"))
    for b, (_, m) in enumerate(rows):
        lp[b, :fl[b], :tl[b]] = m
    dur, _ = _mas_gpu(lp, fl, tl, max(fl), max(tl))
    for b, (d, _) in enumerate(rows):
        assert dur[b, :tl[b]].tolist() == d.tolist()
    from seamless_communication_b200 import ops
    with pytest.raises(RuntimeError, match="8192"):
        z = torch.zeros(1, 2, 8193, device="cuda")
        ops.monotonic_align(z, torch.tensor([2], dtype=torch.int32, device="cuda"),
                            torch.tensor([8193], dtype=torch.int32, device="cuda"))


def _engine_vs_oracle(cfg, sd, text_ids, unit_ids, what):
    """Engine lprob against the float64 oracle on the same weights, element by element within
    oracle_aligner.lprob_error_bound: six standard deviations of the propagated fp16 rounding errors (each rounding an
    independent uniform error, carried through the convs and projected on each distance), plus the fp32 distance and
    softmax roundings.  A rounding-error model rather than a worst case: the worst case, every rounding aligned through
    |W|, is more than 1e5 times the observed error at full width and would guard nothing.
    Durations: the engine's path is the alignment search on its lprob (sb_monotonic_align equals that search bit for bit,
    test_monotonic_align_bit_exact_against_float64).  Wherever the engine's path leaves the oracle's (equal at column
    j + 1, different at j), the oracle's decision there must be a near-tie: |Q[i-1][j] - Q[i][j]| at i = A[j+1] within
    twice the bound on a path score through column j, the sum over columns j' <= j of the largest lprob bound of j' (plus
    the fp32 rounding of the oracle's lprob).  Columns after such a point differ until the paths meet again; they are
    listed with the divergence points."""
    from seamless_communication_b200.aligner_engine import AlignerEngine
    eng = AlignerEngine(cfg, sd)
    lp, dur = eng.forward(text_ids[None], unit_ids[None], [len(text_ids)], [len(unit_ids)])
    lp, dur = lp[0].cpu().double(), dur[0].cpu()
    sd64 = {k: v.double() for k, v in sd.items()}
    te = sd64["alignment_frontend.embed_text.weight"][text_ids]
    ue = sd64["alignment_frontend.embed_unit.weight"][unit_ids]
    P = "alignment_encoder."
    ref, t, f = O.encoder_lprob(sd64, te, ue, cfg.temperature, prefix=P)
    bound = O.lprob_error_bound(f, t, O.state_error_std(sd64, ue, O.FEAT_CONVS, P), O.state_error_std(sd64, te, O.TEXT_CONVS, P),
                                cfg.temperature, ref)
    err = (lp - ref).abs()
    print(f"{what}: max |lprob - lprob64| = {err.max().item():.3e}, max bound {bound.max().item():.3e}, "
          f"largest error / bound {(err / bound).max().item():.3f}")
    assert (err <= bound).all(), (err - bound).max().item()
    path = O.mas_path(lp.float().numpy())
    assert dur.tolist() == np.bincount(path, minlength=len(text_ids)).tolist()
    assert int(dur.sum()) == len(unit_ids)
    ref32 = ref.float().numpy()
    ref_path = O.mas_path(ref32)
    Q = O.mas_q(ref32)
    col_bound = (bound.max(-1).values + O.U32 * ref.abs().max(-1).values).numpy()
    q_bound = 2 * np.cumsum(col_bound)
    differ = np.nonzero(path != ref_path)[0].tolist()
    starts = [j for j in differ if path[j + 1] == ref_path[j + 1]]
    for j in starts:
        i = ref_path[j + 1]
        margin = abs(Q[i - 1, j] - Q[i, j])
        assert margin <= q_bound[j], (what, j, margin, q_bound[j])
    if differ:
        print(f"{what}: paths leave each other at near-tie columns {starts}; differing columns {differ}")
    return lp, dur


@pytest.mark.gpu
def test_engine_tiny_against_the_oracle():
    cfg = C.tiny_aligner()
    sd = S.make_aligner_state_dict(cfg, seed=3)
    g = torch.Generator().manual_seed(2)
    for N, F_ in ((30, 100), (1, 7), (9, 3), (5, 1), (64, 400)):
        text = torch.randint(0, cfg.text_vocab_size, (N,), generator=g)
        units = torch.randint(4, cfg.num_units + 4, (F_,), generator=g)
        _engine_vs_oracle(cfg, sd, text, units, f"tiny_aligner {N}x{F_}")


@pytest.mark.gpu
def test_engine_full_width_500_units_150_characters():
    cfg = C.nar_t2u_aligner()
    sd = S.make_aligner_state_dict(cfg, seed=4)
    g = torch.Generator().manual_seed(3)
    text = torch.randint(4, 40, (150,), generator=g)
    units = torch.randint(4, cfg.num_units + 4, (500,), generator=g)
    _engine_vs_oracle(cfg, sd, text, units, "nar_t2u_aligner 150x500")


@pytest.mark.gpu
def test_ragged_batch_rows_equal_rows_alone():
    from seamless_communication_b200.aligner_engine import AlignerEngine
    cfg = C.tiny_aligner()
    eng = AlignerEngine(cfg, S.make_aligner_state_dict(cfg, seed=6))
    g = torch.Generator().manual_seed(4)
    shapes = [(30, 100), (1, 1), (70, 33), (5, 600), (64, 64), (2, 1)]
    tl, ul = [s[0] for s in shapes], [s[1] for s in shapes]
    tids = torch.full((len(shapes), max(tl)), 10 ** 6)  # padding ids are never looked up
    uids = torch.full((len(shapes), max(ul)), -5)
    for b, (N, F_) in enumerate(shapes):
        tids[b, :N] = torch.randint(0, cfg.text_vocab_size, (N,), generator=g)
        uids[b, :F_] = torch.randint(0, cfg.unit_vocab_size, (F_,), generator=g)
    lp, dur = eng.forward(tids, uids, tl, ul)
    for b, (N, F_) in enumerate(shapes):
        lp1, dur1 = eng.forward(tids[b:b + 1, :N], uids[b:b + 1, :F_], [N], [F_])
        assert torch.equal(lp[b, :F_, :N], lp1[0]), b
        assert torch.equal(dur[b, :N], dur1[0]), b
        assert (dur[b, N:] == 0).all() and (lp[b, F_:] == 0).all() and (lp[b, :F_, N:] == float("-inf")).all()


@pytest.mark.gpu
def test_alignment_extractor_audio_equals_units_and_batch_equals_rows():
    from seamless_communication_b200.models.aligner import AlignmentExtractor
    ex = AlignmentExtractor("tiny_aligner", "tiny_xlsr", 3, None, synthetic=True, num_centroids=256)
    g = torch.Generator().manual_seed(9)
    waves = [0.1 * torch.randn(n, generator=g) for n in (32000, 16001, 8000)]
    texts = ["hello world", "a", "the quick brown fox"]
    rows = []
    for w, txt in zip(waves, texts):
        dur, ids, toks = ex.extract_alignment(w, txt, add_trailing_silence=True)
        units = ex.unit_extractor.predict(w, 2)
        dur_u, ids_u, toks_u = ex.extract_alignment(units, txt, add_trailing_silence=True)
        assert torch.equal(dur, dur_u) and torch.equal(ids, ids_u) and toks == toks_u
        assert dur.dtype == torch.int64 and int(dur.sum()) == len(units) and dur.shape == ids.shape
        assert ex.detokenize_text(ids[0, :-1]) == txt
        rows.append((dur, ids, toks))
    stereo = torch.stack([waves[0], waves[0]])
    assert torch.equal(ex.extract_alignment(stereo, texts[0], add_trailing_silence=True)[0], rows[0][0])
    batch = ex.extract_alignment_batch([waves[0], ex.unit_extractor.predict(waves[1], 2), waves[2]], texts,
                                       add_trailing_silence=True)
    for (d, i, t), (d1, i1, t1) in zip(batch, rows):
        assert torch.equal(d, d1) and torch.equal(i, i1) and t == t1
