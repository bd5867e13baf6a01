"""MinTox (mitigation of added toxicity at inference time): the ETOX word-list check and the re-decode with banned
sequences (reference toxicity/etox_bad_word_checker.py and toxicity/mintox.py)."""
from .etox_bad_word_checker import ETOXBadWordChecker, load_etox_bad_word_checker
from .mintox import mintox_pipeline

__all__ = ["ETOXBadWordChecker", "load_etox_bad_word_checker", "mintox_pipeline"]
