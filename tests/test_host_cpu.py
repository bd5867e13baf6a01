"""CPU-side tests: C-ABI library loads and exports every declared symbol, host logic mirrors the reference's, the
data-parallel plumbing works over gloo with world_size 2.  No kernel is launched here."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from seamless_communication_b200 import _lib, config as C, synthetic as S
from seamless_communication_b200.inference.generator import SequenceGeneratorOptions, remove_consecutive_repeated_ngrams
from seamless_communication_b200.inference.translator import Modality, Task, Translator
from seamless_communication_b200.models.unity.unit_tokenizer import UnitTokenizer
from seamless_communication_b200.nn import PaddingMask, get_seqs_and_padding_mask
from seamless_communication_b200.parallel import shard_bounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")


def test_library_exports_every_header_symbol():
    hdr = open(os.path.join(ROOT, "include", "seamless_b200.h")).read()
    declared = set(re.findall(r"\b(sb_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"sb_stream_t", "sb_gemm_t", "sb_beam_t"}
    lib = _lib.load()
    missing = [n for n in sorted(declared) if not hasattr(lib, n)]
    assert not missing, f"symbols declared in include/seamless_b200.h but not exported: {missing}"
    assert set(_lib.PROTOTYPES) >= declared, sorted(declared - set(_lib.PROTOTYPES))
    assert lib.sb_version() >= 1


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """The drop-in boundary is a C ABI: include/seamless_b200.h compiles as C99 and a C program links against the library."""
    src = tmp_path / "t.c"
    src.write_text('#include "seamless_b200.h"\n'
                   "int main(void) { sb_gemm_t g; sb_resblock_t r; sb_beam_t b; (void)g; (void)r; (void)b;\n"
                   "  return (sb_version() >= 1 && sb_launch_count() >= 0) ? 0 : 1; }\n")
    libdir = os.path.dirname(_lib.LIB_PATH)
    exe = tmp_path / "t"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-lseamless_b200", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([str(exe)]).returncode == 0


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        Translator("seamlessM4T_v2_tiny", "vocoder_v2_tiny", device=torch.device("cpu"))
    with pytest.raises(RuntimeError):
        _lib.require_cuda()


def test_product_package_never_touches_the_oracle_or_the_reference_tree():
    """The oracle is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import it.
    No module of the product package may import `oracle`, shell out to it, or read /root/reference at run time."""
    pkg = os.path.join(ROOT, "seamless_communication_b200")
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if not f.endswith((".py", ".cu", ".cuh", ".h")):
                continue
            src = open(os.path.join(dirpath, f), encoding="utf-8").read()
            if re.search(r"^\s*(from|import)\s+oracle\b", src, re.M) or "oracle/_ref" in src or "libknf_ref" in src \
                    or re.search(r"[\"']/root/reference", src):
                offenders.append(os.path.relpath(os.path.join(dirpath, f), ROOT))
    assert not offenders, offenders
    # and the struct layouts the ctypes binding declares match the header's field lists (same names, same order)
    hdr = open(os.path.join(ROOT, "include", "seamless_b200.h")).read()
    for ctype, cname in ((_lib.GemmDesc, "sb_gemm_t"), (_lib.BeamDesc, "sb_beam_t"), (_lib.ResblockDesc, "sb_resblock_t")):
        body = re.search(r"typedef struct \{([^{}]*)\}\s*" + cname + ";", hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            first, *rest = decl.split(",")
            names.append(re.findall(r"(\w+)\s*(?:\[\d+\])?$", first.strip())[0])
            names += [re.findall(r"(\w+)\s*(?:\[\d+\])?$", r.strip())[0] for r in rest]
        assert names == [f[0] for f in ctype._fields_], (cname, names, [f[0] for f in ctype._fields_])


# ---- streaming policy (a17): pinned against the reference agent -------------------------------------------------------
def _policy_script():
    import importlib.util
    spec = importlib.util.spec_from_file_location("policy_script", os.path.join(G, "policy_script.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _ScriptedModel:
    """decode / project of the monotonic decoder replaced by the deterministic script the fixture generator used."""

    def __init__(self, ps, salt):
        self.ps, self.salt = ps, salt

    def decode(self, ids, encoder_output):
        row = ids[0].tolist()
        logits, probs = self.ps.script(row, int(encoder_output.shape[1]), self.salt)
        dec = torch.zeros(1, len(row), self.ps.VOCAB)
        dec[0, -1] = torch.from_numpy(logits)
        pc = torch.full((self.ps.LAYERS, self.ps.HEADS, len(row), 4), 0.5)
        pc[:, :, -1, -1] = torch.from_numpy(probs)
        return dec, pc

    def project(self, dec):
        return dec


def test_streaming_policy_matches_reference_agent_traces():
    """MMATextDecoderPolicy against call-by-call traces of the reference's MMATextDecoderAgent.policy
    (tests/golden/policy_traces.json, made by tests/golden/make_golden_policy.py): thresholds and decision methods,
    length budget incl. the double-count re-check, burst limit, starting wait, no_early_stop, both n-gram rules."""
    import json
    from seamless_communication_b200.streaming import MMATextDecoderPolicy
    ps = _policy_script()
    traces = json.load(open(os.path.join(G, "policy_traces.json")))
    assert set(traces) == {s["name"] for s in ps.SCENARIOS}
    assert sum(t["ngram_blocks"] for t in traces.values()) >= 20  # the repeat rules are really exercised
    for name, tr in traces.items():
        a = tr["args"]
        pol = MMATextDecoderPolicy(_ScriptedModel(ps, tr["salt"]), prefix=[ps.EOS, 5], eos_idx=ps.EOS,
                                   decision_threshold=a["decision_threshold"], decision_method=a["decision_method"],
                                   p_choose_start_layer=a["p_choose_start_layer"], max_len_a=a["max_len_a"],
                                   max_len_b=a["max_len_b"], max_consecutive_writes=a["max_consecutive_write"],
                                   min_starting_wait=a["min_starting_wait"], no_early_stop=a["no_early_stop"],
                                   block_ngrams=a["block_ngrams"])
        for i, call in enumerate(tr["calls"]):
            new, finished = pol.policy(torch.zeros(1, call["src"], 8), call["final"])
            if call["action"] == "R":
                assert (new, finished) == ([], False), (name, i, new, finished)
            else:
                assert new == call["tokens"] and finished == call["finished"], (name, i, new, call)
        assert pol.target_finished == tr["calls"][-1].get("finished", False), name


def test_streaming_policy_agrees_with_oracle_policy_on_the_oracle_model():
    """The flow of tests/test_gpu_parity.py::test_monotonic_decoder_pchoose_and_policy_match_oracle with the CUDA model
    replaced by the fp32 oracle: product policy and oracle policy take the same decisions given the same model."""
    from oracle.unity_oracle import UnityOracle
    from seamless_communication_b200.streaming import MMATextDecoderPolicy
    cfg = C.tiny_v2()
    sd = S.make_monotonic_state_dict(cfg, seed=2)
    toks = S.make_tokenizers(cfg)
    uo = UnityOracle(cfg.to_dict(), sd, toks)

    class OracleModel:
        def decode(self, ids, enc):
            return uo.monotonic_decoder(ids, enc)

        def project(self, dec):
            return uo.project(dec)

    torch.manual_seed(4)
    enc = torch.randn(1, 13, cfg.model_dim).half().float()
    prefix = [3, toks[0].lang_index("spa")]
    for budget in (10, 3):
        pol = MMATextDecoderPolicy(OracleModel(), prefix=prefix, eos_idx=cfg.text_eos, max_len_a=0, max_len_b=budget)
        written, o_target = [], []
        for n, fin in ((5, False), (9, False), (13, True)):
            new, finished = pol.policy(enc[:, :n], fin)
            o_new, o_fin = uo.emma_policy(enc[:, :n], prefix, o_target, fin, max_len=budget)
            o_target += o_new
            written += new
            assert new == o_new and finished == o_fin, (budget, n, new, o_new, finished, o_fin)
            if finished:
                break
        assert written == o_target and len(written) > 0


def test_unit_tokenizer_matches_reference_kats():
    d = np.load(os.path.join(G, "unit_tokenizer.npz"))
    langs = ["eng", "deu", "fra"]
    for arch in ("nar_multilingual_v2", "base"):
        tk = UnitTokenizer(100, langs, arch)
        assert tk.vocab_info.size == int(d[arch + ".vocab_size"])
        assert [tk.lang_to_index(l) for l in langs] == d[arch + ".lang_index"].tolist()
        assert tk.index_to_lang(tk.lang_to_index("fra")) == "fra"
        enc = tk.create_encoder("deu")
        assert np.array_equal(enc(torch.from_numpy(d[arch + ".enc_in"])).numpy(), d[arch + ".enc_out"])
        dec = tk.create_decoder()
        assert np.array_equal(dec(torch.from_numpy(d[arch + ".dec_in"])).numpy(), d[arch + ".dec_out"])
    with pytest.raises(ValueError):
        UnitTokenizer(100, langs, "base").lang_to_index("xyz")
    with pytest.raises(ValueError):
        UnitTokenizer(100, langs, "base").create_encoder("xyz")
    # vocabulary sizes of the reference's own unit test (tests/unit/models/unity/test_unity.py:24,41)
    assert UnitTokenizer(100, langs, "base").vocab_info.size == 112
    assert UnitTokenizer(100, langs, "nar_multilingual_v2").vocab_info.size == 108


def test_ngram_filter_and_options_defaults():
    import json
    for c in json.load(open(os.path.join(G, "ngram_filter.json"))):  # outputs of the reference's own function
        assert remove_consecutive_repeated_ngrams(list(c["seq"]), c["min_size"], c["max_size"]) == c["out"]
    assert remove_consecutive_repeated_ngrams([1, 2, 2, 3]) == [1, 2, 3]
    assert remove_consecutive_repeated_ngrams([1, 2, 3, 1, 2, 3, 4]) == [1, 2, 3, 4]
    assert remove_consecutive_repeated_ngrams([]) == []
    o = SequenceGeneratorOptions()
    assert (o.beam_size, o.soft_max_seq_len, o.hard_max_seq_len, o.unk_penalty, o.len_penalty) == (5, (1, 200), 1024, 0.0, 1.0)


def test_vocoder_facade_argument_handling_matches_reference():
    """Vocoder.forward's language / speaker resolution against the reference's own Vocoder.forward
    (tests/golden/vocoder_facade.json), with a recording stand-in for the CUDA engine."""
    import json
    from seamless_communication_b200.models.vocoder.vocoder import Vocoder
    seen = []
    voc = Vocoder(lambda units, lang, spkr: seen.append((list(units.shape), lang, spkr)), C.vocoder_lang_spkr_idx_map())
    for c in json.load(open(os.path.join(G, "vocoder_facade.json"))):
        voc(torch.zeros(c["units_shape"], dtype=torch.int64), c["lang"], c["spkr"], dur_prediction=False)
        shape, lang, spkr = seen[-1]
        assert shape == c["seen"]["code_shape"] and lang == c["seen"]["lang"] and spkr == c["seen"]["spkr"], c
    with pytest.raises(KeyError):
        voc(torch.zeros(2, 3, dtype=torch.int64), "xxx", -1, dur_prediction=False)
    with pytest.raises(NotImplementedError):
        voc(torch.zeros(2, 3, dtype=torch.int64), "eng", -1, dur_prediction=True)


def test_task_routing_and_padding_mask():
    assert Translator.get_modalities_from_task_str("s2st") == (Modality.SPEECH, Modality.SPEECH)
    assert Translator.get_modalities_from_task_str("S2TT") == (Modality.SPEECH, Modality.TEXT)
    assert Translator.get_modalities_from_task_str("asr") == (Modality.SPEECH, Modality.TEXT)
    assert Translator.get_modalities_from_task_str("t2tt") == (Modality.TEXT, Modality.TEXT)
    assert Translator.get_modalities_from_task_str("t2st") == (Modality.TEXT, Modality.SPEECH)
    with pytest.raises(ValueError):
        Translator.get_modalities_from_task_str("s2x")
    assert [t.name for t in Task] == ["S2ST", "S2TT", "T2ST", "T2TT", "ASR"]
    m = PaddingMask(torch.tensor([3, 1]), 4)
    assert m.materialize().tolist() == [[True, True, True, False], [True, False, False, False]]
    assert m.trim(1).seq_lens.tolist() == [2, 0] and m.trim(1).batch_seq_len == 3
    seqs, mask = get_seqs_and_padding_mask({"seqs": torch.zeros(2, 4, 80), "seq_lens": torch.tensor([4, 2]), "is_ragged": True})
    assert mask is not None and mask.seq_lens.tolist() == [4, 2]
    assert get_seqs_and_padding_mask({"seqs": torch.zeros(2, 4), "seq_lens": torch.tensor([4, 4]), "is_ragged": False})[1] is None


def test_synthetic_assets_follow_reference_layout():
    cfg = C.tiny_v2()
    tok, ctok = S.make_tokenizers(cfg)
    assert tok.vocab_info.size == cfg.text_vocab and (tok.vocab_info.pad_idx, tok.vocab_info.unk_idx, tok.vocab_info.eos_idx) == (0, 1, 3)
    enc = tok.create_encoder(task="translation", lang="spa", mode="target")
    assert enc.prefix_indices.tolist() == [3, tok.lang_index("spa")]  # [</s>, __spa__] (ggml_convert.py:131-135)
    src = tok.create_encoder(lang="eng", mode="source")
    ids = src("aaab aaac").tolist()
    assert ids[0] == tok.lang_index("eng") and ids[-1] == 3
    assert tok.create_decoder()(torch.tensor(ids)) == "aaab aaac"
    with pytest.raises(ValueError):
        tok.create_encoder(lang="xxx")
    sd = S.make_unity_state_dict(cfg, 0)
    # names a maintainer would recognise from convert_unity_checkpoint (models/unity/loader.py:206-386)
    for k in ("speech_encoder.inner.layers.0.self_attn.sdpa.rel_k_embed.weight", "speech_encoder.adaptor_layers.0.residual_conv.weight",
              "text_decoder.layers.1.encoder_decoder_attn.q_proj.weight", "t2u_model.decoder.layers.0.conv1d.conv1.weight",
              "t2u_model.decoder_frontend.variance_adaptor.duration_predictor.conv1.0.weight", "final_proj.weight"):
        assert k in sd
    assert sd["final_proj.weight"] is sd["text_decoder_frontend.embed.weight"]  # TiedProjection (builder.py:451)
    assert sd["speech_encoder.inner.layers.0.conv.depthwise_conv.weight"].shape == (cfg.model_dim, 1, 31)
    full = C.base_v2()
    assert (full.model_dim, full.enc_layers, full.dec_layers, full.text_vocab, full.unit_vocab, full.char_vocab) == \
           (1024, 24, 24, 256102, 10082, 10943)


def test_decode_splits_keep_the_step_slices():
    """The K slices of a decoder step's split-K products fix its fp32 sums and so its search results: q|k|v, the three
    model_dim x model_dim products and FFN out, for the 1024 / 8192 models (base, base_v2, small_*) and tiny_* (128 / 256)."""
    from seamless_communication_b200.ops import decode_splits
    want = {(1024, 8192): {5: (2, 8, 8), 40: (2, 8, 8), 160: (2, 8, 8), 161: (2, 4, 8), 256: (2, 4, 8), 257: (2, 4, 8)},
            (128, 256): {5: (1, 2, 1), 40: (1, 2, 1), 160: (1, 2, 1), 161: (1, 1, 1), 256: (1, 1, 1), 257: (1, 1, 1)}}
    for (dim, ffn), by_rows in want.items():
        for rows, splits in by_rows.items():
            assert decode_splits(rows, dim, ffn) == splits, (dim, ffn, rows)


def test_shard_bounds_cover_batch():
    for n, w in ((256, 8), (33, 4), (3, 8)):
        spans = [shard_bounds(n, w, r) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from seamless_communication_b200.parallel import scatter_batch, gather_padded, shard_bounds
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
g = torch.arange(6 * 5, dtype=torch.float32).view(6, 5) if rank == 0 else None
mine = scatter_batch(g, 3, (5,), torch.float32, "cpu")
lo, hi = shard_bounds(6, 2, rank)
assert torch.equal(mine, torch.arange(6 * 5, dtype=torch.float32).view(6, 5)[lo:hi]), mine
# ranks produce different output lengths (rank r: 4 + r samples per row)
out = mine[:, :1].repeat(1, 4 + rank) + rank
outs, lens = gather_padded(out, torch.full((3,), 4 + rank, dtype=torch.int64))
if rank == 0:
    assert [o.shape for o in outs] == [torch.Size([3, 4]), torch.Size([3, 5])], [o.shape for o in outs]
    assert torch.equal(outs[1][:, 0], torch.arange(6 * 5, dtype=torch.float32).view(6, 5)[3:, 0] + 1)
    assert lens[1].tolist() == [5, 5, 5]
dist.barrier()
dist.destroy_process_group()
print("ok", rank)
"""


def test_scatter_gather_world_size_2_gloo(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    port = str(29500 + (os.getpid() % 2000))
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True) for r in range(2)]
    outs = [p.communicate(timeout=120)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs


# ------------------------------------------------------------------------------------------------ checkpoint ingestion (8f.3)
def test_checkpoint_conversion_matches_reference_functions():
    """models/checkpoint.py against the mapping produced by EXECUTING the reference's own _fairseq_key_map /
    convert_unity_checkpoint / _get_char_index_mapping / convert_vocoder_checkpoint (tests/golden/make_golden_keymap.py):
    every example key (one per rule of the reference's table) is renamed identically, the converted state dict has the same
    keys, and the rewritten tensors (control-symbol row permutation, NLLB dummy row, tied tables, character permutation)
    are identical."""
    import json
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import make_golden_keymap as mk
    from seamless_communication_b200.models import checkpoint as ck
    fx = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "unity_keymap.json")))
    assert len(fx["patterns"]) >= 90
    for old, new in fx["rename"].items():
        if new is not None:
            assert ck.rename_key(old) == new, (old, new, ck.rename_key(old))
    sd = mk.make_inputs({p: None for p in fx["patterns"]})
    out = ck.convert_unity_checkpoint({"model": sd}, char_pieces=fx["char_pieces"])["model"]
    assert sorted(out.keys()) == fx["output_keys"]
    for k, c in fx["checksums"].items():
        assert mk.checksum(out[k]) == c, k
    assert out["text_decoder_frontend.embed.weight"] is out["final_proj.weight"]          # one tied table
    assert out["t2u_model.decoder_frontend.embed.weight"] is out["t2u_model.final_proj.weight"]
    assert ck.char_index_mapping(fx["char_pieces"]) == fx["char_index_mapping"]
    assert sorted(ck.convert_vocoder_checkpoint({"generator": {"conv_pre.weight_g": 1, "ups.0.bias": 2}})["model"]) == fx["vocoder_keys"]
    # a checkpoint already in fairseq2 naming passes through
    done = {"model": {"speech_encoder.inner.layers.0.self_attn_layer_norm.weight": torch.zeros(1)}}
    assert ck.convert_unity_checkpoint(done)["model"] is done["model"]


def test_model_loaders_refuse_to_invent_weights():
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.models.vocoder import load_vocoder_model
    with pytest.raises(RuntimeError, match="synthetic=True"):
        load_unity_model("seamlessM4T_v2_large", device="cpu")
    with pytest.raises(RuntimeError, match="synthetic=True"):
        load_vocoder_model("vocoder_v2", device="cpu")


def test_lane_pool_host_logic():
    """parallel.LanePool without a GPU: every lane is one thread bound to one engine lane, jobs of a lane run in
    submission order, results come back in order, a failing job (or a failing lane set-up) surfaces through its future."""
    import threading
    import time
    from seamless_communication_b200.parallel import LanePool

    class FakeEngine:
        def __init__(self):
            self.tls = threading.local()

        def set_lane(self, i):
            self.tls.lane = i

    eng = FakeEngine()
    pool = LanePool("cpu", 3, [eng])
    log = []

    def job(i):
        time.sleep(0.01 * (5 - i % 5))  # later jobs finish earlier unless the lane serialises them
        log.append((eng.tls.lane, i))
        return eng.tls.lane, i

    try:
        outs = pool.map(job, [(i,) for i in range(9)])
        assert outs == [(i % 3, i) for i in range(9)]  # round-robin lanes, results in submission order
        for lane in range(3):
            assert [i for l, i in log if l == lane] == [lane, lane + 3, lane + 6]  # in-lane order kept
        pool.warm(job, 0)
        with pytest.raises(ZeroDivisionError):
            pool.submit(1, lambda: 1 // 0).result(timeout=10)
        assert pool.submit(1, lambda: 7).result(timeout=10)[0] == 7  # the lane survives a failed job
    finally:
        pool.close()

    class BrokenEngine:
        def set_lane(self, i):
            raise RuntimeError("no such lane")

    pool = LanePool("cpu", 1, [BrokenEngine()])
    try:
        with pytest.raises(RuntimeError, match="no such lane"):
            pool.submit(0, lambda: 1).result(timeout=10)
    finally:
        pool.close()


def test_evaluate_driver_files_order_and_corrupted_inputs(tmp_path):
    """seamless_communication_b200.evaluate.run_eval (the reference's cli/m4t/evaluate driver, evaluate.py:116-366) with a
    stub translator: manifest parsing (TSV + JSON lines), WAV decoding (PCM16 / float32 / stereo), buckets in file order,
    undecodable and NaN inputs replaced by the reference's dummy outputs, a RuntimeError batch skipped, output files."""
    import json
    import wave as wave_mod
    from pathlib import Path
    from seamless_communication_b200 import evaluate as E
    from seamless_communication_b200.inference.translator import BatchedSpeechOutput

    audio = tmp_path / "audio"
    audio.mkdir()
    g = torch.Generator().manual_seed(0)
    lengths = [16000, 12000, 8000, 20000, 4000, 6000, 10000]
    for i, n in enumerate(lengths):
        x = torch.rand(n, generator=g) * 0.5 - 0.25
        if i == 1:  # stereo PCM16 through the standard library writer: channel 0 is used
            with wave_mod.open(str(audio / f"{i}.wav"), "wb") as w:
                w.setnchannels(2); w.setsampwidth(2); w.setframerate(16000)
                st = torch.stack([x, -x], dim=1)
                w.writeframes((st * 32767).round().to(torch.int16).numpy().tobytes())
        elif i == 2:
            x[100] = float("nan")
            E.write_wav_f32(audio / f"{i}.wav", x)
        elif i == 4:
            (audio / f"{i}.wav").write_bytes(b"not a wav file")
        else:
            E.write_wav_f32(audio / f"{i}.wav", x)
    got = E.decode_wav(audio / "1.wav")
    assert got.shape == (12000,) and got.abs().max() <= 0.25 + 1e-3
    assert E.decode_wav(audio / "4.wav") is None and E.decode_wav(audio / "missing.wav") is None
    back = E.decode_wav(audio / "0.wav")
    assert back.shape == (16000,) and back.dtype == torch.float32

    tsv = tmp_path / "dev.tsv"
    tsv.write_text("id\taudio\ttgt_text\n" + "".join(f"{i}\t{i}.wav\tref {i}\n" for i in range(len(lengths))))

    class StubTranslator:
        device = torch.device("cpu")
        calls = []

        def fbank_batch(self, batch, lens):
            return {"seqs": batch, "seq_lens": lens, "is_ragged": True}

        def predict(self, src, task, tgt_lang, **kw):
            lens = src["seq_lens"].tolist()
            self.calls.append(lens)
            if 20000 in lens:
                raise RuntimeError("The sequence generator returned no hypothesis at index 0. Please file a bug report.")
            assert src["seqs"].shape == (len(lens), max(lens)) and task == "s2st" and tgt_lang == "spa"
            return ([f"hyp {n}" for n in lens],
                    BatchedSpeechOutput(units=[[n % 7, 3] for n in lens], audio_wavs=[torch.full((1, 1, n // 10), 0.5) for n in lens]))

    ctx = E.EvalContext(task="s2st", data_file=tsv, audio_root_dir=audio, target_lang="spa", output_path=tmp_path / "out", batch_size=2)
    tr = StubTranslator()
    res = E.run_eval(tr, ctx, lanes=2)
    # buckets: (0,1) ok | (2 NaN,3 -> RuntimeError batch skipped) | (4 undecodable, 5) | (6)
    assert sorted(map(tuple, tr.calls)) == sorted([(16000, 12000), (20000,), (6000,), (10000,)])
    assert res["samples"] == 5 and res["skipped"] == 2 and res["corrupted"] == 2
    lines = res["model_outputs"].read_text().splitlines()
    assert lines[0] == "ref_tgt_text\tpred_tgt_text\tpred_tgt_audio"
    body = [l.split("\t") for l in lines[1:]]
    assert [b[:2] for b in body] == [["ref 0", "hyp 16000"], ["ref 1", "hyp 12000"], ["ref 4", ""], ["ref 5", "hyp 6000"],
                                      ["ref 6", "hyp 10000"]]
    units = res["unit_outputs"].read_text().splitlines()
    assert units == ["5 3", "2 3", "", "1 3", "4 3"]
    wavs = [E.decode_wav(Path(b[2])) for b in body]
    assert [w.numel() for w in wavs] == [1600, 1200, 16000, 600, 1000]  # the dummy is one second of silence
    assert wavs[2].abs().max() == 0 and abs(float(wavs[0][0]) - 0.5) < 1e-6
    assert [Path(b[2]).name for b in body] == [f"{i}_pred.wav" for i in range(5)]

    # JSON-lines manifest (m4t_prepare_dataset layout), text output only
    js = tmp_path / "dev.json"
    js.write_text("".join(json.dumps({"source": {"text": "s", "lang": "eng", "audio_local_path": f"{i}.wav"},
                                      "target": {"text": f"ref {i}"}}) + "\n" for i in (0, 5)))

    class TextStub(StubTranslator):
        def predict(self, src, task, tgt_lang, **kw):
            return [f"hyp {n}" for n in src["seq_lens"].tolist()], None

    from seamless_communication_b200.inference.translator import Modality
    ctx2 = E.EvalContext(task="s2tt", data_file=js, audio_root_dir=audio, target_lang="spa", output_path=tmp_path / "out",
                         output_modality=Modality.TEXT, batch_size=4)
    res2 = E.run_eval(TextStub(), ctx2)
    assert res2["model_outputs"].read_text().splitlines() == ["ref_tgt_text\tpred_tgt_text", "ref 0\thyp 16000", "ref 5\thyp 6000"]
    with pytest.raises(NotImplementedError):
        E.run_eval(TextStub(), E.EvalContext(task="t2tt", data_file=js, audio_root_dir=audio, target_lang="spa",
                                             output_path=tmp_path / "out", input_modality=Modality.TEXT))
