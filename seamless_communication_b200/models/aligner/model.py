"""UnitY2 forced aligner model (reference models/aligner/model.py:25-304, builder.py, loader.py) on `AlignerEngine`.

Deviations from the reference (DESIGN.md section 12): fp16 weights and activations with fp32 accumulation whatever the
caller's dtype; fp32 distances and log-softmax; the alignment search's first row is a float64 running sum where numpy
sums the float32 row pairwise (they differ only by rounding); rows of a batch are each computed as the row alone; only
reduction_factor 1.
"""
from __future__ import annotations

from typing import Any, List, Mapping, Optional, Tuple, Union

import torch
from torch import Tensor

from ... import config as cfgmod
from ... import synthetic as synthetic_mod
from ...aligner_engine import AlignerEngine
from ..unity.unit_tokenizer import UnitTokenizer


class UnitY2AlignmentFrontend:
    """Tokenisation of the aligner's two inputs (model.py:25-71): characters through the character model's raw encoding
    (`synthetic.RawCharEncoder` over the tokenizer's piece model, i.e. `synthetic.char_pieces`), units through the card's
    UnitTokenizer with `is_nar_decoder` forced on (u + 4, ids >= num_units + 4 become unk).  The embeddings themselves
    live in the engine."""

    def __init__(self, cfg: cfgmod.AlignerConfig, char_tokenizer) -> None:
        self.text_tokenizer = char_tokenizer
        self.unit_tokenizer = UnitTokenizer(cfg.num_units, list(cfg.unit_langs), cfg.name)
        self.unit_tokenizer.is_nar_decoder = True
        self.encode_text = synthetic_mod.RawCharEncoder(char_tokenizer.model, char_tokenizer.vocab_info.unk_idx)
        self.encode_unit = self.unit_tokenizer.create_encoder(lang="eng")

    def tokenize_text(self, text: str, add_trailing_silence: bool = False) -> Tensor:
        ids = self.encode_text(text)
        return torch.cat([ids, ids[0:1]]) if add_trailing_silence else ids

    def tokenize_text_to_tokens(self, text: str, add_trailing_silence: bool = False) -> List[str]:
        toks = self.encode_text.encode_as_tokens(text)
        return toks + toks[:1] if add_trailing_silence else toks

    def tokenize_unit(self, units: Union[str, Tensor]) -> Tensor:
        if isinstance(units, str):
            units = torch.tensor([int(u) for u in units.split(" ")])
        return self.encode_unit(units)

    def decode_text(self, ids: Tensor) -> str:
        """SentencePiece decoding of character ids: pad / bos / eos are dropped, unk reads " ⁇ ", "▁" is a space
        and the leading one is removed."""
        vi = self.text_tokenizer.vocab_info
        out = []
        for i in torch.as_tensor(ids).reshape(-1).tolist():
            if i in (vi.pad_idx, vi.bos_idx, vi.eos_idx):
                continue
            out.append(" ⁇ " if i == vi.unk_idx else self.text_tokenizer.model.index_to_token(int(i)))
        s = "".join(out).replace(synthetic_mod.SPACE, " ")
        return s[1:] if s.startswith(" ") else s


class UnitY2AlignmentModel:
    alignment_frontend: UnitY2AlignmentFrontend
    engine: AlignerEngine

    def __init__(self, cfg: cfgmod.AlignerConfig, frontend: UnitY2AlignmentFrontend, engine: AlignerEngine) -> None:
        self.cfg, self.alignment_frontend, self.engine = cfg, frontend, engine

    def __call__(self, input_text: Tensor, input_unit: Tensor) -> Tuple[Tensor, Tensor]:
        return self.forward(input_text, input_unit)

    def forward(self, input_text: Tensor, input_unit: Tensor) -> Tuple[Tensor, Tensor]:
        """(B, T_text) character ids and (B, T_feat) unit ids, every row full length (model.py:293-304) -> attn_lprob
        (B, T_feat, T_text) fp32 and durations (B, T_text) int64."""
        if input_text.dim() != 2 or input_unit.dim() != 2:
            raise ValueError("input_text and input_unit must be 2-D (batch, length)")
        B = input_text.shape[0]
        return self.engine.forward(input_text, input_unit, [input_text.shape[1]] * B, [input_unit.shape[1]] * B)


def load_unity2_alignment_model(name: str, device="cuda", *, state_dict: Optional[Mapping[str, Tensor]] = None,
                                checkpoint: Union[str, Mapping[str, Any], None] = None, synthetic: bool = False, seed: int = 5,
                                char_tokenizer=None) -> UnitY2AlignmentModel:
    """name: "nar_t2u_aligner" (the card) or the test copy "tiny_aligner" (config.ALIGNER_ARCHS).  Weights come from
    `state_dict` (reference names), `checkpoint` (path or mapping of `unity2_aligner.pt`, converted by
    models/checkpoint.py `convert_unity2_aligner_checkpoint`) or `synthetic=True` (seeded random init); without any a
    RuntimeError is raised.  char_tokenizer: the card's character model (an object with `model.index_to_token`,
    `model.token_to_index` and `vocab_info`, e.g. synthetic.SyntheticCharTokenizer); text is encoded from its pieces by
    `synthetic.char_pieces`.  Only a synthetic model may go without one."""
    if name not in cfgmod.ALIGNER_ARCHS:
        raise ValueError(f"unknown aligner '{name}' (known: {sorted(cfgmod.ALIGNER_ARCHS)})")
    cfg = cfgmod.ALIGNER_ARCHS[name]()
    if char_tokenizer is None:
        if not synthetic or state_dict is not None or checkpoint is not None:
            raise RuntimeError(f"no character tokenizer for '{name}': pass char_tokenizer=... (the card's SentencePiece "
                               "model cannot be downloaded here)")
        char_tokenizer = synthetic_mod.SyntheticCharTokenizer(cfg.text_vocab_size)
    if state_dict is None and checkpoint is not None:
        from ..checkpoint import convert_unity2_aligner_checkpoint, load_checkpoint_file
        ck = load_checkpoint_file(checkpoint) if isinstance(checkpoint, str) else checkpoint
        pieces = [char_tokenizer.model.index_to_token(i) for i in range(char_tokenizer.vocab_info.size)]
        state_dict = convert_unity2_aligner_checkpoint(ck, pieces)["model"]
    if state_dict is None:
        if not synthetic:
            raise RuntimeError(f"no weights for '{name}': pass state_dict=..., checkpoint=... or synthetic=True")
        state_dict = synthetic_mod.make_aligner_state_dict(cfg, seed=seed)
    frontend = UnitY2AlignmentFrontend(cfg, char_tokenizer)
    return UnitY2AlignmentModel(cfg, frontend, AlignerEngine(cfg, dict(state_dict), device=device))
