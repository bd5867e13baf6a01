"""Programmatic dependent launch (PDL, common.cuh) changes when kernels start, never what they compute: with it (the
default) and without it (SB_PDL=0) the same seeded work gives the same bits.  The setting is read once per process, so
each setting runs in a child process of its own (this file run as a script) and the parent compares what they saved:
  - a beam search on `small_v2` at 32 sentences x beam 5 (160 rows) over 102 positions: its hypotheses, the device
    search state (seqs, scores, finished hypotheses) and the harvested decoder states; the same search on 2 lanes and
    with banned sequences;
  - Translator.predict(..., "s2st") on the tiny config: texts, unit ids, waveforms;
  - the weight-stationary products (decode_gemm_kernel) at every wgmma width, at K slices shorter and longer than the
    ring, and the vocabulary projection (vocab_proj_kernel) at a K of 2 k-blocks and of 16: bit-identical to the
    row-major kernels in each process, and across the two."""
import hashlib
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dev = "cuda"
HARD_MAX = 102


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def _search_record(eng, hyps):
    st = eng._last_search_state
    fin = st["fin"]
    lengths = [len(h[0][1]) - 1 for h in hyps]
    harvested = eng.harvest_decoder_states(lengths)
    return dict(hyps=hyps, seqs=st["seqs"].cpu(), scores=st["scores"].cpu(),
                fin={k: v.cpu() for k, v in fin.items() if isinstance(v, torch.Tensor)},
                harvested=harvested.buf.cpu())


def _encoder_input(cfg, seed, B=32, S_enc=13):
    from seamless_communication_b200.ops import Seq
    g = torch.Generator(device=dev).manual_seed(seed)
    e = Seq(B, S_enc, cfg.model_dim, buf=torch.randn(B * S_enc, cfg.model_dim, device=dev, generator=g).half())
    lens = torch.randint(3, S_enc + 1, (B,), dtype=torch.int32, device=dev, generator=g)
    lens[0] = S_enc
    return e, lens


def _searches():
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.parallel import LanePool
    eng = load_unity_model("small_v2", synthetic=True, seed=7, dec_gain=4.0).engine
    prefix = [eng.cfg.text_eos, eng.text_tokenizer.lang_index("spa")]

    def search(seed, banned=None):
        e, lens = _encoder_input(eng.cfg, seed)
        hyps = eng.beam_search(e, lens, prefix, beam=5, soft_max=(1, 200), hard_max=HARD_MAX, banned=banned)
        torch.cuda.synchronize()
        return _search_record(eng, hyps)

    out = dict(plain=search(23))
    # bans that bite: the first generated token of the longest best hypothesis, and its next two tokens as a pair
    best = max((h[0][1] for h in out["plain"]["hyps"]), key=len)
    assert len(best) >= 5, best
    out["banned_seqs"] = [[best[2]], best[3:5]]
    out["banned"] = search(23, banned=out["banned_seqs"])
    pool = LanePool("cuda", 2, [eng])
    try:
        pool.warm(search, 23)
        futs = [pool.submit(i, search, 31 + i) for i in range(2)]
        out["lanes"] = [f.result()[0] for f in futs]
    finally:
        pool.close()
    return out


def _s2st():
    from seamless_communication_b200 import config as C, synthetic as S
    from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    cfg, vc = C.tiny_v2(), C.tiny_vocoder()
    model = load_unity_model("tiny_v2", state_dict=S.make_unity_state_dict(cfg, 0, dec_gain=4.0, dur_gain=1.0, dur_bias=0.9),
                             tokenizers=S.make_tokenizers(cfg))
    voc = load_vocoder_model("tiny", state_dict=S.make_vocoder_state_dict(vc, 1))
    tr = Translator(model, voc, device=dev)
    opts = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=24)
    texts, speech = tr.predict(tr.fbank_batch(S.make_waveforms(3, 32000, seed=5).to(dev)), "s2st", "spa",
                               text_generation_opts=opts)
    torch.cuda.synchronize()
    return dict(texts=texts, units=speech.units, wavs=[a.float().cpu() for a in speech.audio_wavs])


def _products():
    """Partials of the transposed kernel at every row width class (wgmma N 32 / 64 / 128 / 160 / 256) and at split counts
    whose K slices are shorter than the ring (1024 x 1024 at 8 and 16 slices: 2 and 1 k-blocks, ring >= 2) and longer
    (1 and 2 slices of q|k|v: 16 and 8 k-blocks); FFN inner in direct mode (16 k-blocks); the projection at 16 k-blocks
    (a ring of 5 at 160 rows) and at 2.  Each against the row-major kernels at the same slices."""
    from seamless_communication_b200 import ops
    from seamless_communication_b200.ops import Seq
    M, FFN = 1024, 8192
    out, mismatches = {}, []
    g = torch.Generator(device=dev).manual_seed(3)
    for rows in (5, 37, 128, 160, 256):
        SR = ops.slice_rows(rows)
        a = Seq(1, rows, M, buf=torch.randn(rows, M, device=dev, generator=g).half())
        for n, k, splits in ((3 * M, M, (1, 2, 4)), (M, M, (1, 2, 4, 8, 16)), (M, FFN, (8, 32))):
            ak = a if k == M else Seq(1, rows, k, buf=torch.randn(rows, k, device=dev, generator=g).half())
            w = (torch.randn(n, k, device=dev, generator=g) / math.sqrt(k)).half()
            for s in splits:
                want, got = (torch.zeros(s * SR, n, device=dev) for _ in range(2))
                ops.gemm_splitk(ak, w, n, s, want)
                ops.gemm_splitk(ak, w, n, s, got, transposed=True)
                got = got.view(s, SR, n)[:, :rows]
                if not torch.equal(got, want.view(s, SR, n)[:, :rows]):
                    mismatches.append(("splitk", rows, n, k, s))
                out[("splitk", rows, n, k, s)] = _digest(got)
        w = (torch.randn(FFN, M, device=dev, generator=g) / math.sqrt(M)).half()
        bias = torch.randn(FFN, device=dev, generator=g)
        want = ops.gemm(a, w, FFN, bias, act=ops.ACT_RELU, out=Seq(1, rows, FFN))
        got = ops.gemm_decode(a, w, FFN, bias, act=ops.ACT_RELU, out=Seq(1, rows, FFN))
        if not torch.equal(got.buf, want.buf):
            mismatches.append(("direct", rows))
        out[("direct", rows)] = _digest(got.buf)
    for R, V, k in ((160, 256102, M), (37, 256102, M), (160, 3001, 128)):
        a = Seq(1, R, k, buf=torch.randn(R, k, device=dev, generator=g).half())
        w = (torch.randn(V, k, device=dev, generator=g) * 0.05).half()
        res = []
        for proj_t in ("1", "0"):
            os.environ["SB_PROJ_T"] = proj_t
            logits = Seq(1, R, V, dtype=torch.float32, buf=torch.full((R, (V + 7) // 8 * 8), float("nan"), device=dev))
            stats = torch.full(((V + 127) // 128, R, 2), float("nan"), device=dev)
            ops.gemm(a, w, V, None, out=logits, out_f32=True, tile_stats=stats)
            res.append((logits.buf[:, :V].clone(), stats))
        del os.environ["SB_PROJ_T"]
        if not (torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])):
            mismatches.append(("proj", R, V, k))
        out[("proj", R, V, k)] = (_digest(res[0][0]), _digest(res[0][1]))
    return dict(digests=out, mismatches=mismatches)


def _child(path):
    from seamless_communication_b200 import _lib
    torch.save(dict(pdl=_lib.load().sb_pdl_enabled(), products=_products(), searches=_searches(), s2st=_s2st()), path)


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("pdl")
    res = {}
    for name, setting in (("default", None), ("off", "0")):
        env = {k: v for k, v in os.environ.items() if k != "SB_PDL"}
        if setting is not None:
            env["SB_PDL"] = setting
        path = d / f"{name}.pt"
        subprocess.run([sys.executable, "-s", os.path.abspath(__file__), str(path)], env=env, cwd=ROOT, check=True, timeout=1800)
        res[name] = torch.load(path, weights_only=False)
    assert res["default"]["pdl"] == 1 and res["off"]["pdl"] == 0
    return res


def _assert_same_search(a, b):
    assert a["hyps"] == b["hyps"]
    for key in ("seqs", "scores", "harvested"):
        assert torch.equal(a[key], b[key]), key
    assert a["fin"].keys() == b["fin"].keys()
    for key in a["fin"]:
        assert torch.equal(a["fin"][key], b["fin"][key]), key


def test_search_is_bit_identical_with_and_without_pdl(runs):
    _assert_same_search(runs["default"]["searches"]["plain"], runs["off"]["searches"]["plain"])


def test_banned_search_is_bit_identical_with_and_without_pdl(runs):
    d, o = runs["default"]["searches"], runs["off"]["searches"]
    assert d["banned_seqs"] == o["banned_seqs"]
    assert d["banned"]["hyps"] != d["plain"]["hyps"]  # the bans changed the search
    _assert_same_search(d["banned"], o["banned"])


def test_two_lane_searches_are_bit_identical_with_and_without_pdl(runs):
    for a, b in zip(runs["default"]["searches"]["lanes"], runs["off"]["searches"]["lanes"]):
        _assert_same_search(a, b)


def test_s2st_is_bit_identical_with_and_without_pdl(runs):
    d, o = runs["default"]["s2st"], runs["off"]["s2st"]
    assert d["texts"] == o["texts"] and d["units"] == o["units"]
    assert len(d["wavs"]) == len(o["wavs"])
    for x, y in zip(d["wavs"], o["wavs"]):
        assert torch.equal(x, y)


def test_weight_stationary_products_match_row_major_with_and_without_pdl(runs):
    d, o = runs["default"]["products"], runs["off"]["products"]
    assert d["mismatches"] == [] and o["mismatches"] == []
    assert d["digests"] == o["digests"]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    _child(sys.argv[1])
