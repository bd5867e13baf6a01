"""ETOX added-toxicity check (behavioural mirror of reference toxicity/etox_bad_word_checker.py).

A target text has added toxicity when it contains words of its language's ETOX list and the source text contains none
of the source language's.  Words match as whole space-delimited words of the lower-cased text with every non-word
character turned into a space; for the card's SentencePiece languages they match as a contiguous run of SentencePiece
tokens instead."""
from __future__ import annotations

import codecs
import os
import re
from typing import Any, Dict, Iterable, List, Optional

from .. import config as cfgmod


class ETOXBadWordChecker:
    """`bad_words[lang]`: the language's word list; `bad_word_variants[lang][word]`: the spellings banned when `word`
    is found (lower, upper and capitalized); `sp_encoder.encode_as_tokens(text)`: the SentencePiece tokens of a text,
    used for the languages in `sp_langs`."""

    def __init__(self, bad_words: Dict[str, List[str]], bad_word_variants: Dict[str, Dict[str, List[str]]],
                 sp_encoder: Optional[Any], sp_langs: Iterable[str]):
        self.bad_words = bad_words
        self.bad_word_variants = bad_word_variants
        self.sp_encoder = sp_encoder
        self.sp_langs = set(sp_langs)

    def extract_bad_words(self, source_text: str, target_text: str, source_lang: str, target_lang: str) -> List[str]:
        """The variants of every word found in `target_text`, or [] when none is found there or when `source_text`
        already holds one of its own language's words (the toxicity was not added by the translation)."""
        found = self.get_bad_words(target_text, target_lang)
        if not found or self.get_bad_words(source_text, source_lang):
            return []
        variants = self.bad_word_variants[target_lang]
        return [v for word in found for v in variants[word]]

    def get_bad_words(self, text: str, lang: str) -> List[str]:
        if lang not in self.bad_words:
            raise RuntimeError(f"MinTox model does not support {lang}.")
        words = self.bad_words[lang]
        text = re.sub(r"[\W+]", " ", text.lower())
        if lang in self.sp_langs:
            if self.sp_encoder is None:
                raise RuntimeError(f"checking {lang} needs the SentencePiece encoder (sp_encoder) of the MinTox card")
            tokens = list(self.sp_encoder.encode_as_tokens(text.lower()))
            return [str(w) for w in words if _has_run(tokens, list(self.sp_encoder.encode_as_tokens(w.lower())))]
        padded = f" {text.lower()} "
        return [w.lower().strip(" ") for w in words if f" {w.lower()} " in padded]


def _has_run(tokens: List[Any], run: List[Any]) -> bool:
    n = len(run)
    return any(tokens[i:i + n] == run for i in range(len(tokens) - n + 1))


def _file_lang(name: str) -> str:
    return name[:8] if name[:8] in cfgmod.MINTOX_ETOX_LANG_VARIANTS else name[:3]


def _read_words(path: str) -> List[str]:
    """One rot13-encoded word per line; duplicates dropped (first occurrence kept, so the order is reproducible)."""
    with open(path, "r", encoding="utf-8") as f:
        words = [codecs.decode(line, "rot_13").rstrip("\n") for line in f.readlines()]
    return list(dict.fromkeys(words))


def load_etox_bad_word_checker(model_name_or_card: str = "mintox", *, dataset_dir: Optional[str] = None,
                               sp_encoder: Optional[Any] = None) -> ETOXBadWordChecker:
    """The `mintox` card's checker from a local copy of its ETOX dataset (the NLLB-200 toxicity word lists, one rot13
    file per language).  Nothing is downloaded: `dataset_dir` is required.  `sp_encoder` (anything with
    `encode_as_tokens(text)`, e.g. fairseq2's SentencePieceEncoder over the card's `sp_model`) is needed only to check the
    card's SentencePiece languages.  A file's language is its name's first 8 characters when that is one of the card's
    language variants, otherwise its first 3; files are read in name order."""
    if model_name_or_card != "mintox":
        raise ValueError(f"unknown toxicity card {model_name_or_card!r}; the ETOX checker belongs to 'mintox'")
    if dataset_dir is None:
        raise ValueError("load_etox_bad_word_checker needs dataset_dir: the directory of the card's ETOX word lists "
                         "(nllb-200_twl.zip, unpacked); this implementation downloads nothing")
    bad_words: Dict[str, List[str]] = {}
    variants: Dict[str, Dict[str, List[str]]] = {}
    for name in sorted(os.listdir(dataset_dir)):
        path = os.path.join(dataset_dir, name)
        if not os.path.isfile(path):
            continue
        lang = _file_lang(name)
        words = _read_words(path)
        bad_words[lang] = words
        variants[lang] = {w: [w.lower(), w.upper(), w.capitalize()] for w in words}
    return ETOXBadWordChecker(bad_words, variants, sp_encoder, cfgmod.MINTOX_SP_LANGS)
