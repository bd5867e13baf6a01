#!/usr/bin/env python
"""Generates tests/golden/vocoder_36langs_map.json: the language / speaker table of the reference's vocoder_36langs
asset card (src/seamless_communication/cards/vocoder_36langs.yaml, `model_config.lang_spkr_idx_map`), the vocoder of
seamlessM4T_large.

Run from the repo root (needs /root/reference; the GPU box only reads the committed fixture):

    python tests/golden/make_golden_vocoder36.py

The card's model_config is a JSON object inside the YAML file; it is read as JSON, so no YAML parser is needed.
"""
import json
import os

CARD = "/root/reference/src/seamless_communication/cards/vocoder_36langs.yaml"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "vocoder_36langs_map.json")


def main():
    text = open(CARD).read()
    head, body = text.split("model_config:", 1)
    assert "model_arch: base" in head
    cfg = json.loads(body)
    with open(OUT, "w") as f:
        json.dump({"model_arch": "base", "lang_spkr_idx_map": cfg["lang_spkr_idx_map"]}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
