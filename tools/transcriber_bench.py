#!/usr/bin/env python
"""Transcriber stage timings on the synthetic seamlessM4T_v2_large: B utterances of L seconds, beam 1 (DESIGN.md section 13).

Per stage, medians of --reps calls timed with CUDA events (host-side stages with a host clock after a synchronise):
  * encoder (fbank batch included);
  * the search with and without recording the attention, alternated call by call, so the per-step cost of
    sb_decode_cross_attn_weights shows as their difference;
  * sb_token_timestamps on the recorded search;
  * the host word grouping;
  * the reference's post-processing arm: the winners' attention copied to the host, then per row numpy normalisation,
    scipy.signal.medfilt2d and an O(F^2) pure-Python longest increasing subsequence (the cost profile of
    inference/transcriber.py:178-235);
  * transcribe_batch against a loop of transcribe over the same inputs.
The card's name and power limit are printed from the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.signal import medfilt2d  # noqa: E402


def reference_postprocess(A: np.ndarray, width: int):
    """inference/transcriber.py's _extract_timestamps cost profile on one row's (n, F) matrix (restated)."""
    A = A / A.sum(axis=0, keepdims=1)
    A = medfilt2d(A, kernel_size=(width, width))
    c = np.argmax(A, axis=0)
    arr = [(int(k), -j) for j, k in enumerate(c)]
    n = len(arr)
    L, prev = [1] * n, list(range(n))
    for i in range(1, n):
        for j in range(i):
            if arr[i] > arr[j] and L[i] < L[j] + 1:
                L[i], prev[i] = L[j] + 1, j
    return L, prev


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop-rows", type=int, default=8, help="rows of the transcribe_batch / transcribe-loop comparison")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transcriber_bench.py needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else torch.cuda.get_device_name()
    print("card:", card)
    from seamless_communication_b200 import synthetic as S
    from seamless_communication_b200.inference import Transcriber
    tr = Transcriber("seamlessM4T_v2_large", "cuda", synthetic=True)
    eng = tr.engine
    n_samp = int(a.seconds * 16000)
    waves = S.make_waveforms(a.batch, n_samp, seed=3)
    prefix = tr.tokenizer.create_encoder(task="translation", lang="eng", mode="target").prefix_indices.tolist()
    opts = dict(beam=1, soft_max=(1, 128), hard_max=1024)
    holder = {}

    def encode():
        f = tr._frontend.fbank_batch(waves)
        holder["enc"], holder["lens"] = eng.encode_speech(f["seqs"].half().contiguous(), None)

    encode()
    enc = holder["enc"]
    for rec in (False, True, False, True):  # warm-up: both graphs captured
        eng.beam_search(enc, None, prefix, record_attention=rec, **opts)
    t_enc = timed(encode, a.reps)
    plain, record, steps = [], [], []
    for _ in range(a.reps):
        for rec, dst in ((False, plain), (True, record)):
            dst.append(timed(lambda: eng.beam_search(enc, None, prefix, record_attention=rec, **opts), 1))
            if rec:
                steps.append(int(eng._last_search_state["step"].item()))
    t_plain, t_rec = statistics.median(plain), statistics.median(record)
    hyps = eng.beam_search(enc, None, prefix, record_attention=True, **opts)
    t_ts_call = timed(lambda: eng.token_timestamps(3), a.reps)
    stamps = eng.token_timestamps(3)
    # the kernel alone, on the buffers the call above builds
    from seamless_communication_b200 import _lib
    st = eng._last_search_state
    sel, n = eng._best_hypotheses(st)
    slots = st["fin"]["anc"][torch.arange(a.batch, device="cuda"), sel].contiguous()
    n_dev = torch.tensor(n, dtype=torch.int32, device="cuda")
    per_row = max(max(n), 1) * (enc.T - 2)
    scratch = torch.empty((a.batch, per_row), dtype=torch.float64, device="cuda")
    starts = torch.zeros((a.batch, max(max(n), 1)), dtype=torch.int32, device="cuda")
    lib = _lib.load()
    t_ts = timed(lambda: lib.sb_token_timestamps(st["attn_hist"].data_ptr(), st["R"], enc.T, slots.data_ptr(), slots.stride(0),
                                                 n_dev.data_ptr(), None, len(prefix), a.batch, 3, scratch.data_ptr(), per_row,
                                                 starts.data_ptr(), starts.shape[1], torch.cuda.current_stream().cuda_stream), a.reps)
    F = enc.T - 2
    pieces = [[tr.tokenizer.model.index_to_token(i) for i in h[0][1][len(prefix):-1]] for h in hyps]
    t0 = time.perf_counter()
    for b in range(a.batch):
        per = a.seconds / F
        Transcriber._collect_word_level_stats(pieces[b], [per * s for s in stamps[b][0]], stamps[b][1])
    t_words = (time.perf_counter() - t0) * 1e3
    n_tok = [len(s[0]) for s in stamps]

    def reference_arm():
        A, n = eng.harvest_attention()
        A = A.double().cpu().numpy()
        for b in range(a.batch):
            if n[b]:
                reference_postprocess(A[b, :n[b], 1:1 + F], 3)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    reference_arm()
    t_ref = (time.perf_counter() - t0) * 1e3
    rows = [waves[i] for i in range(min(a.loop_rows, a.batch))]
    tr.transcribe_batch(rows, "eng")
    tr.transcribe(rows[0], "eng")
    t_batch = timed(lambda: tr.transcribe_batch(rows, "eng"), max(1, a.reps // 2))
    t_loop = timed(lambda: [tr.transcribe(w, "eng") for w in rows], max(1, a.reps // 2))
    res = dict(card=card, batch=a.batch, seconds=a.seconds, encoder_frames=enc.T, tokens_mean=float(np.mean(n_tok)),
               search_steps=statistics.median(steps), encoder_ms=t_enc, search_ms=t_plain, search_recording_ms=t_rec,
               recording_per_step_us=(t_rec - t_plain) / max(1, statistics.median(steps)) * 1e3,
               sb_token_timestamps_ms=t_ts, token_timestamps_call_ms=t_ts_call, word_grouping_ms=t_words, reference_postprocess_ms=t_ref,
               reference_postprocess_per_row_ms=t_ref / a.batch, loop_rows=len(rows), transcribe_batch_ms=t_batch,
               transcribe_loop_ms=t_loop)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
