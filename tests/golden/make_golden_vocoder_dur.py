#!/usr/bin/env python
"""Generates tests/golden/codehifigan_dur_tiny.npz: the reference's CodeGenerator.forward with dur_prediction=True.

Run from the repo root (needs /root/reference; the GPU box only reads the committed fixture):

    python tests/golden/make_golden_vocoder_dur.py

The reference's own src/seamless_communication/models/vocoder/{hifigan,codehifigan}.py and
models/unity/length_regulator.py (VariancePredictor) run through the shims of make_golden.py, on the tiny vocoder arch
with the synthetic weights of `make_vocoder_state_dict(..., dur_predictor=True)`.

Two cases:
  * "one": N=1, 17 units;
  * "two": N=2, the same unit row twice with different language / speaker.  Rows with equal totals are the only
    multi-row batch the reference can run (torch.cat of the repeat-interleaved rows, codehifigan.py:85-88).
Stored per case: units, lang, spkr, the predictor's exp(l) - 1 before rounding, the durations and the waveform.  The unit
row is the first seeded draw whose every exp(l) - 1 lies at least 0.05 from a half-integer, so that fp16 device
arithmetic cannot round a duration the other way.
"""
import importlib
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import install_shims  # noqa: E402

U = 17
MARGIN = 0.05


def main():
    install_shims()
    from seamless_communication_b200 import config as C, synthetic as S

    lr = importlib.import_module("seamless_communication.models.unity.length_regulator")
    sys.modules["seamless_communication.models.unity"].VariancePredictor = lr.VariancePredictor
    chg = importlib.import_module("seamless_communication.models.vocoder.codehifigan")

    vc = C.tiny_vocoder()
    vsd = S.make_vocoder_state_dict(vc, seed=1, dur_predictor=True)
    dur_params = {"encoder_embed_dim": vc.embedding_dim, "var_pred_hidden_dim": vc.var_pred_hidden,
                  "var_pred_kernel_size": vc.var_pred_kernel, "var_pred_dropout": 0.5}
    gen = chg.CodeGenerator(list(vc.upsample_rates), list(vc.upsample_kernel_sizes), vc.upsample_initial_channel,
                            list(vc.resblock_kernel_sizes), [list(d) for d in vc.resblock_dilation_sizes],
                            vc.model_in_dim, vc.num_embeddings, vc.embedding_dim, dur_params, vc.lang_embedding_dim,
                            vc.num_langs, vc.spkr_embedding_dim, vc.num_spkrs)
    gen.load_state_dict({k[len("code_generator."):]: v for k, v in vsd.items()}, strict=True)
    gen.eval()

    def raw_durations(units):
        with torch.inference_mode():
            return torch.exp(gen.dur_predictor(gen.dict(units), None)) - 1

    for seed in range(1000):
        units = torch.randint(0, vc.num_embeddings, (1, U), generator=torch.Generator().manual_seed(seed))
        raw = raw_durations(units)
        if float(((raw - raw.floor()) - 0.5).abs().min()) >= MARGIN:
            break
    else:
        raise RuntimeError("no unit row with every duration away from a rounding boundary")
    out = {"seed": np.array(seed)}
    for name, u, lang, spkr in (("one", units, [25], [45]), ("two", units.repeat(2, 1), [25, 8], [45, 3])):
        raw = raw_durations(u)
        with torch.inference_mode():
            wav = gen({"code": u, "spkr": torch.tensor(spkr)[:, None], "lang": torch.tensor(lang)[:, None]}, True)
        dur = torch.clamp(torch.round(raw).long(), min=1)
        assert wav.shape == (u.shape[0], 1, int(dur[0].sum()) * vc.hop)
        out.update({f"{name}.units": u.numpy(), f"{name}.lang": np.array(lang), f"{name}.spkr": np.array(spkr),
                    f"{name}.raw": raw.numpy(), f"{name}.dur": dur.numpy(), f"{name}.wav": wav.numpy()})
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "codehifigan_dur_tiny.npz")
    np.savez_compressed(path, **out)
    d = out["one.dur"][0]
    print(f"wrote {path}: unit seed {seed}, durations {d.tolist()} (total {d.sum()})")


if __name__ == "__main__":
    main()
