#!/usr/bin/env python
"""Cost of MinTox at the bench shape: S2ST on seamlessM4T_v2_large + vocoder_v2 with seeded random-init weights, a batch
of 32 x 10 s synthetic utterances, beam 5, hard_max_seq_len 102.

1. The select half of one search step (CUDA-graph replay), without bans (g_sel: top-K, sb_beam_step, sb_step_advance)
   and with 30, 300 and 3000 banned sequences of 1-3 tokens (g_sel_ban: sb_ban_step first).  CUDA events around each
   replay; the step index is reset to the same mid-search position before every replay, outside the timed window.
2. Translator.predict end to end (host clock around a device synchronise): MinTox off, on with no row flagged (the
   check only), and on with 4 of the rows flagged, each by a word only its text holds (the check and a re-decode of
   those rows; the number flagged is printed).

Medians over --iters runs after one warm-up run.  Prints the card's name and power limit."""
import argparse
import codecs
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from seamless_communication_b200 import config as C, synthetic as S  # noqa: E402
from seamless_communication_b200.inference import SequenceGeneratorOptions, Translator  # noqa: E402
from seamless_communication_b200.models.unity import load_unity_model  # noqa: E402
from seamless_communication_b200.models.vocoder import load_vocoder_model  # noqa: E402
from seamless_communication_b200.toxicity import load_etox_bad_word_checker  # noqa: E402
from seamless_communication_b200.toxicity.mintox import _extract_bad_words_with_batch_indices  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--replays", type=int, default=200)
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card)
cfg, vc = C.base_v2(), C.base_vocoder()
toks = S.make_tokenizers(cfg)
model = load_unity_model("seamlessM4T_v2_large", device="cuda", state_dict=S.make_unity_state_dict(cfg, seed=0, dec_gain=4.0),
                         tokenizers=toks)
voc = load_vocoder_model("vocoder_v2", device="cuda", state_dict=S.make_vocoder_state_dict(vc, seed=1))
opts = SequenceGeneratorOptions(beam_size=5, soft_max_seq_len=(1, 200), hard_max_seq_len=102)
plain = Translator(model, voc, device="cuda")
src = plain.fbank_batch(S.make_waveforms(args.batch, 160000, seed=1234).cuda())
texts, _ = plain.predict(src, "s2st", "spa", text_generation_opts=opts)
eng = model.engine
st = eng._last_search_state
prefix = [cfg.text_eos, toks[0].lang_index("spa")]

# ---- 1. select half per step
g = torch.Generator().manual_seed(0)


def random_bans(n):
    return [torch.randint(4, cfg.text_vocab - 300, (1 + j % 3,), generator=g).tolist() for j in range(n)]


def time_select(graph):
    ts = []
    for _ in range(args.replays):
        st["step"].fill_(40)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        ts.append((e0, e1))
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) * 1e3 for a, b in ts)


with torch.inference_mode():
    eng._search_reset(st, prefix)
    print(f"select per step, {st['R']} rows (us, median of {args.replays}):")
    print(f"  no bans (g_sel)      {time_select(st['g_sel']):8.1f}")
    for n in (30, 300, 3000):
        eng._set_bans(st, random_bans(n))
        if st["g_sel_ban"] is None:
            eng._capture_ban(st)
        eng._search_reset(st, prefix)
        time_select(st["g_sel_ban"])  # warm-up
        print(f"  {n:5d} banned seqs     {time_select(st['g_sel_ban']):8.1f}   (table capacity {st['ban']['cap']})")

# ---- 2. predict end to end
tmp = tempfile.mkdtemp()


def checker(tgt_words, src_words=("zzzzqq",)):
    """ETOX lists for spa (target) and eng (source)."""
    d = os.path.join(tmp, str(len(os.listdir(tmp))))
    os.mkdir(d)
    for name, ws in (("spa_twl.txt", tgt_words), ("eng_twl.txt", src_words)):
        with open(os.path.join(d, name), "w", encoding="utf-8") as f:
            f.write("".join(codecs.encode(w, "rot_13") + "\n" for w in ws))
    return load_etox_bad_word_checker("mintox", dataset_dir=d)


# four rows are flagged, each by a word that no other row's text holds (the source texts are the first pass's texts)
rows_of = {}
for i, t in enumerate(texts):
    for w in set(t.split()):
        rows_of.setdefault(w, []).append(i)
unique = {}
for w, r in sorted(rows_of.items()):
    if len(r) == 1:
        unique.setdefault(r[0], w)
flag_checker = checker([unique[i] for i in sorted(unique)[:4]] or ["zzzzqq"])
n_flagged = len(_extract_bad_words_with_batch_indices(texts, texts, "eng", "spa", flag_checker)[1])
runs = [("apply_mintox off", plain),
        ("on, nothing flagged", Translator(model, voc, device="cuda", apply_mintox=True, bad_word_checker=checker(["zzzzqq"]))),
        (f"on, {n_flagged} rows flagged", Translator(model, voc, device="cuda", apply_mintox=True, bad_word_checker=flag_checker))]


def predict(tr):
    return tr.predict(src, "s2st", "spa", src_lang="eng", text_generation_opts=opts)


print(f"Translator.predict, S2ST {args.batch} x 10 s (ms, median of {args.iters}):")
for name, tr in runs:
    predict(tr)
    ts = []
    for _ in range(args.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out_texts, _ = predict(tr)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    changed = sum(a != b for a, b in zip(out_texts, texts))
    print(f"  {name:22s} {statistics.median(ts):8.1f}   rows whose text changed: {changed}")
