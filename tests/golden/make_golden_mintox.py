#!/usr/bin/env python
"""Generates tests/golden/mintox_etox.json by driving the REFERENCE's ETOX checker and MinTox helpers
(src/seamless_communication/toxicity/etox_bad_word_checker.py and mintox.py, imported from /root/reference) over a
synthetic rot13 word-list dataset, and records the mintox card's `etox_lang_variants` / `sp_langs`
(src/seamless_communication/cards/mintox.yaml).  fairseq2 is absent offline: the types the two modules import are
stand-ins defined below; the card, the asset store and the download manager are fakes that hand the real
ETOXBadWordCheckerLoader the synthetic dataset and the card's own field values.

    python tests/golden/make_golden_mintox.py
"""
import codecs
import importlib.util
import json
import os
import sys
import tempfile
import types
from pathlib import Path

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SEAMLESS_REF", "/root/reference")
OUT = os.path.join(HERE, "mintox_etox.json")

# word lists, one file per language.  Names cover the card's language variants (kept whole), a variant-like name that is
# not one (cut to 3 letters), a SentencePiece language, and words repeated within a file.
WORDS = {
    "spa_twl.txt": ["abcd", "efgh ijkl", "Mnop", "abcd", "qrst"],
    "eng_twl.txt": ["uvwx", "qrst", "uvwx"],
    "zho_Hans_twl.txt": ["yzab", "cdef"],
    "zho_Hant_twl.txt": ["ghij"],
    "knc_Latx_twl.txt": ["klmn"],
    "hin_twl.txt": ["abcdef", "opqr", "xy"],
    "fra_twl.txt": ["Mnop"],
}


class StubSpEncoder:
    """A SentencePiece stand-in: each space-delimited word becomes "▁" + its first two letters, then two-letter pieces."""

    def encode_as_tokens(self, text):
        out = []
        for w in str(text).split():
            out.append("▁" + w[:2])
            out += [w[i:i + 2] for i in range(2, len(w), 2)]
        return out


def dataset_files():
    return {name: "".join(codecs.encode(w, "rot_13") + "\n" for w in words) for name, words in WORDS.items()}


def card_fields():
    import yaml
    card = yaml.safe_load(open(os.path.join(REF, "src/seamless_communication/cards/mintox.yaml")))
    return card["etox_lang_variants"], card["sp_langs"]


def install_shims():
    def mod(name, **attrs):
        m = sys.modules.get(name) or types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    ph = type("Placeholder", (), {})

    class SentencePieceModel:
        def __init__(self, path):
            self.path = path

    class SentencePieceEncoder(StubSpEncoder):
        def __init__(self, model):
            self.model = model

    class BannedSequenceProcessor:
        def __init__(self, seqs):
            self.seqs = seqs

    mod("fairseq2")
    mod("fairseq2.assets", AssetCard=type("AssetCard", (), {}), AssetDownloadManager=ph, AssetStore=ph, asset_store=None,
        download_manager=None)
    mod("fairseq2.data", StringLike=str, SequenceData=dict)
    mod("fairseq2.data.text", SentencePieceEncoder=SentencePieceEncoder, SentencePieceModel=SentencePieceModel)
    mod("fairseq2.data.text.text_tokenizer", TextTokenizer=ph)
    mod("fairseq2.data.typing", StringLike=str)
    mod("fairseq2.typing", Device=ph)
    mod("fairseq2.generation", BannedSequenceProcessor=BannedSequenceProcessor)
    mod("fairseq2.nn")
    mod("fairseq2.nn.padding", get_seqs_and_padding_mask=None)
    mod("seamless_communication").__path__ = [os.path.join(REF, "src/seamless_communication")]
    mod("seamless_communication.inference", SequenceGeneratorOptions=ph)
    mod("seamless_communication.models")
    mod("seamless_communication.models.unity", UnitTokenizer=ph, UnitYModel=ph)
    mod("seamless_communication.toxicity").__path__ = [os.path.join(REF, "src/seamless_communication/toxicity")]


def load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, "src/seamless_communication", rel))
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def main():
    install_shims()
    etox = load("seamless_communication.toxicity.etox_bad_word_checker", "toxicity/etox_bad_word_checker.py")
    mintox = load("seamless_communication.toxicity.mintox", "toxicity/mintox.py")
    variants, sp_langs = card_fields()
    files = dataset_files()
    with tempfile.TemporaryDirectory() as d:
        for name, text in files.items():
            open(os.path.join(d, name), "w", encoding="utf-8").write(text)

        class Field:
            def __init__(self, v):
                self.v = v

            def as_set(self, _):
                return set(self.v)

            def as_uri(self):
                return self.v

        class Card:
            name = "mintox"

            def field(self, k):
                return Field({"etox_lang_variants": variants, "sp_langs": sp_langs, "etox_dataset": "etox://local",
                              "sp_model": "sp://local"}[k])

        class Downloads:
            def download_dataset(self, uri, name):
                return Path(d)

            def download_tokenizer(self, uri, name):
                return Path(d) / "sp.model"

        class Store:
            def retrieve_card(self, name):
                assert name == "mintox"
                return Card()

        checker = etox.ETOXBadWordCheckerLoader(Store(), Downloads())("mintox")
    out = dict(etox_lang_variants=variants, sp_langs=sp_langs, files=files,
               bad_words={k: sorted(v) for k, v in checker.bad_words.items()},
               bad_word_variants={k: {w: v for w, v in sorted(m.items())} for k, m in checker.bad_word_variants.items()})
    get_cases = [("abcd, qrst!", "spa"), ("xabcd qrstx", "spa"), ("EFGH   ijkl", "spa"), ("efgh-ijkl", "spa"),
                 ("mnop", "spa"), ("efgh", "spa"), ("", "spa"), ("YZAB.", "zho_Hans"), ("ghij", "zho_Hant"),
                 ("klmn", "knc"), ("abcdef", "hin"), ("abcdefgh", "hin"), ("zzab cdef", "hin"), ("x opqr", "hin"),
                 ("xyz", "hin"), ("uvwx", "eng")]
    out["get_bad_words"] = [[t, l, sorted(checker.get_bad_words(t, l))] for t, l in get_cases]
    extract_cases = [("hello", "hello there", "eng", "spa"),           # nothing in the target
                     ("uvwx", "abcd here", "eng", "spa"),              # the source has its own word
                     ("clean", "abcd and efgh ijkl", "eng", "spa"),    # added toxicity
                     ("clean", "Mnop", "fra", "spa"),                  # found lower-cased, listed capitalised
                     ("clean", "abcdef", "eng", "hin")]
    ext = []
    for s, t, sl, tl in extract_cases:
        try:
            ext.append([s, t, sl, tl, sorted(checker.extract_bad_words(s, t, sl, tl)), None])
        except Exception as e:  # noqa: BLE001 - the fixture records the reference's exception
            ext.append([s, t, sl, tl, None, f"{type(e).__name__}: {e}"])
    out["extract_bad_words"] = ext
    try:
        checker.get_bad_words("abcd", "xyz")
        raise AssertionError("expected an error")
    except RuntimeError as e:
        out["unsupported_error"] = str(e)
    srcs, tgts = ["a", "b", "uvwx", "d"], ["abcd", "none here", "qrst", "efgh ijkl qrst"]
    words, idx = mintox._extract_bad_words_with_batch_indices(srcs, tgts, "eng", "spa", checker)
    out["batch_indices"] = dict(src=srcs, tgt=tgts, words=sorted(words), indices=idx)
    texts = ["t0", "t1", "t2", "t3", "t4"]
    mintox._replace_with_new_text_output_in_batch(texts, [1, 3], ["n1", "n3"])
    out["replace_text"] = dict(indices=[1, 3], new=["n1", "n3"], result=texts)
    unit_tok = types.SimpleNamespace(vocab_info=types.SimpleNamespace(pad_idx=1))
    cases = []
    for width_new in (3, 5, 7):
        orig = torch.arange(20, dtype=torch.int64).reshape(4, 5) + 10
        new = torch.arange(2 * width_new, dtype=torch.int64).reshape(2, width_new) + 100
        o0 = orig.clone()
        ret = mintox._replace_with_new_unit_output_in_batch(unit_tok, orig, torch.tensor([0, 2]), new)
        cases.append(dict(original=o0.tolist(), new=new.tolist(), indices=[0, 2], returned=ret,
                          original_after=orig.tolist()))
    out["replace_units"] = cases
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, ensure_ascii=False)
        f.write("\n")


if __name__ == "__main__":
    main()
