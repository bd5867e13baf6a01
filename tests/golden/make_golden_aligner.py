#!/usr/bin/env python
"""Generates tests/golden/aligner.npz by EXECUTING the reference's own aligner code here (needs the reference tree;
nothing is copied).  fairseq2 is replaced by type-only stand-ins, except `to_padding_mask`, whose one line of behaviour
(position < length) is restated; at batch 1 every position is valid, so it masks nothing here.

  * `_aligner_nar_t2u` (models/aligner/builder.py:64-87): every config field, and `num_units` / `unit_langs` of
    cards/nar_t2u_aligner.yaml;
  * `UnitY2AlignmentEncoder` (model.py:79-190) built in float64 at width 16 from seeded weights: its state-dict names and
    shapes, and its forward (lprob, durations) at batch 1 for several (T_text, T_feat), including T_feat < T_text,
    T_text = 1 and T_feat = 1;
  * `_monotonic_alignment_search` (model.py:212-243) on crafted matrices: exact ties, -inf entries, planted blocks;
  * `convert_unity2_aligner_checkpoint` (loader.py:22-74) on a small seeded checkpoint, with a stand-in char tokenizer
    whose pieces are not in sorted order;
  * `UnitY2AlignmentFrontend.tokenize_unit` (model.py:63-66) through the reference's unit_tokenizer.py, with ids >=
    num_units.
"""
import os
import sys
import types
from dataclasses import asdict

import numpy as np
import torch

REF = "/root/reference/src/seamless_communication"
HERE = os.path.dirname(os.path.abspath(__file__))
WIDTH = 16
ENCODER_CASES = ((1, 7, 9), (2, 5, 5), (3, 8, 3), (4, 1, 6), (5, 6, 1), (6, 1, 1), (7, 12, 40))  # (seed, T_text, T_feat)


def encoder_state_dict(seed: int):
    """float64 weights of UnitY2AlignmentEncoder(WIDTH, WIDTH, 2, 3) under its own names."""
    g = torch.Generator().manual_seed(7000 + seed)
    sd = {}
    for name, k in (("t_conv.1", 3), ("t_conv.4", 1), ("f_conv.1", 3), ("f_conv.4", 3), ("f_conv.7", 1)):
        sd[name + ".weight"] = torch.randn(WIDTH, WIDTH, k, generator=g, dtype=torch.float64) / (WIDTH * k) ** 0.5
        sd[name + ".bias"] = 0.1 * torch.randn(WIDTH, generator=g, dtype=torch.float64)
    return sd


def encoder_inputs(seed: int, T_text: int, T_feat: int):
    g = torch.Generator().manual_seed(8000 + seed)
    return (torch.randn(1, T_text, WIDTH, generator=g, dtype=torch.float64),
            torch.randn(1, T_feat, WIDTH, generator=g, dtype=torch.float64))


def mas_cases():
    """Crafted (T_feat, T_text) log-probability matrices (float32)."""
    cases = {}
    cases["ties"] = np.full((6, 3), -1.0, np.float32)  # every path scores alike: ties everywhere
    m = np.log(np.full((8, 4), 0.25, np.float32))
    m[2, 1] = -np.inf
    m[5, :2] = -np.inf
    cases["neg_inf"] = m.astype(np.float32)
    rng = np.random.default_rng(3)
    dur = [3, 1, 5, 2, 4]
    lp = np.log(rng.uniform(0.01, 0.05, size=(sum(dur), len(dur)))).astype(np.float32)
    j = 0
    for i, d in enumerate(dur):
        lp[j:j + d, i] = np.log(0.9)
        j += d
    cases["planted"] = lp
    cases["short"] = np.log(rng.uniform(0.1, 1, size=(2, 5))).astype(np.float32)  # T_feat < T_text
    cases["one_text"] = np.log(rng.uniform(0.1, 1, size=(5, 1))).astype(np.float32)
    cases["one_feat"] = np.log(rng.uniform(0.1, 1, size=(1, 4))).astype(np.float32)
    cases["random"] = np.log(rng.dirichlet(np.ones(9), size=30)).astype(np.float32)
    return cases


def converter_case():
    """Seeded checkpoint in the aligner's training layout, and a char vocabulary whose pieces are not sorted."""
    g = torch.Generator().manual_seed(9)
    pieces = ["<unk>", "<s>", "</s>", "<pad>", "z", "b", "▁", "a", "y", "c"]
    ck = {"text_emb_state": {"weight": torch.randn(len(pieces) + 2, 4, generator=g)},
          "unit_emb_state": {"weight": torch.randn(12, 4, generator=g)},
          "aligner_state": {"t_conv.1.weight": torch.randn(4, 4, 3, generator=g), "t_conv.1.bias": torch.randn(4, generator=g),
                            "f_conv.7.weight": torch.randn(4, 4, 1, generator=g)}}
    return ck, pieces


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _load(name, path):
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


class _Generic:
    def __class_getitem__(cls, item):
        return cls

    def __init__(self, *args, **kw):
        self.args, self.kw = args, kw


class _Registry(_Generic):
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.archs = {}

    def decorator(self, name):
        return lambda f: self.archs.setdefault(name, f)


class _VocabularyInfo:
    def __init__(self, size, unk_idx, bos_idx, eos_idx, pad_idx):
        self.size, self.unk_idx, self.bos_idx, self.eos_idx, self.pad_idx = size, unk_idx, bos_idx, eos_idx, pad_idx


class _CharTokenizer:
    def __init__(self, pieces):
        self.model = types.SimpleNamespace(index_to_token=lambda i: pieces[i], vocabulary_size=len(pieces))

    def create_raw_encoder(self):
        return None

    def create_decoder(self):
        return None


def load_reference():
    for name in ("fairseq2", "fairseq2.data", "fairseq2.nn", "fairseq2.models", "fairseq2.models.utils", "fairseq2.data.text",
                 "seamless_communication", "seamless_communication.models", "seamless_communication.models.unity",
                 "seamless_communication.models.aligner"):
        _stub(name)
    sys.modules["fairseq2.data"].CString = str
    sys.modules["fairseq2.data"].VocabularyInfo = _VocabularyInfo
    _stub("fairseq2.data.typing", StringLike=str)
    _stub("fairseq2.data.vocabulary_info", VocabularyInfo=_VocabularyInfo)
    _stub("fairseq2.nn.embedding", StandardEmbedding=torch.nn.Embedding, init_scaled_embedding=None)
    _stub("fairseq2.nn.padding", to_padding_mask=lambda lens, n: torch.arange(n, device=lens.device)[None, :] < lens[:, None])
    _stub("fairseq2.typing", DataType=torch.dtype, Device=torch.device)
    _stub("fairseq2.assets", asset_store=None, download_manager=None)
    _stub("fairseq2.assets.card", AssetCard=object)
    _stub("fairseq2.models.utils", ConfigLoader=_Generic, ModelLoader=_Generic)
    _stub("fairseq2.models.utils.arch_registry", ArchitectureRegistry=_Registry)
    state = {}
    _stub("seamless_communication.models.unity.char_tokenizer", CharTokenizer=object,
          load_unity_char_tokenizer=lambda card: state["char_tokenizer"])
    _stub("seamless_communication.models.unity.loader", load_unity_unit_tokenizer=None)
    ut = _load("seamless_communication.models.unity.unit_tokenizer", os.path.join(REF, "models", "unity", "unit_tokenizer.py"))
    model = _load("seamless_communication.models.aligner.model", os.path.join(REF, "models", "aligner", "model.py"))
    builder = _load("seamless_communication.models.aligner.builder", os.path.join(REF, "models", "aligner", "builder.py"))
    loader = _load("seamless_communication.models.aligner.loader", os.path.join(REF, "models", "aligner", "loader.py"))
    return ut, model, builder, loader, state


def card():
    import yaml
    with open(os.path.join(REF, "cards", "nar_t2u_aligner.yaml")) as f:
        return yaml.safe_load(f)


def main():
    ut, model, builder, loader, state = load_reference()
    fx = {}
    cfg = builder.aligner_archs.archs["nar_t2u_aligner"]()
    enc, fe = cfg.alignment_encoder_config, cfg.alignment_frontend_config
    for k, v in asdict(enc).items():
        fx[f"arch.{k}"] = np.array(v)
    vi = fe.unit_vocab_info
    for k in ("size", "unk_idx", "bos_idx", "eos_idx", "pad_idx"):
        fx[f"arch.unit_vocab.{k}"] = np.array(getattr(vi, k))
    fx["arch.text_vocab_size"] = np.array(fe.text_vocab_size)
    fx["arch.model_name_or_card"] = np.array(cfg.model_name_or_card)
    c = card()
    fx["card.num_units"] = np.array(c["num_units"])
    fx["card.unit_langs"] = np.array(c["unit_langs"])
    fx["card.model_arch"] = np.array(c["model_arch"])

    # the encoder at batch 1, float64
    torch.manual_seed(0)
    e = model.UnitY2AlignmentEncoder(WIDTH, WIDTH, 2, 3, 0.1, 1.0, 1, torch.float64).eval()
    names = list(e.state_dict())
    fx["encoder.keys"] = np.array(names)
    fx["encoder.shapes"] = np.array([",".join(map(str, e.state_dict()[k].shape)) for k in names])
    for seed, T_text, T_feat in ENCODER_CASES:
        e.load_state_dict(encoder_state_dict(seed))
        t, f = encoder_inputs(seed, T_text, T_feat)
        with torch.no_grad():
            lp, dur = e(t, f, torch.tensor([T_text]), torch.tensor([T_feat]))
        fx[f"encoder.{seed}.lprob"] = lp[0].numpy()
        fx[f"encoder.{seed}.durations"] = dur[0].numpy()

    for name, m in mas_cases().items():
        fx[f"mas.{name}.lprob"] = m
        fx[f"mas.{name}.path"] = model._monotonic_alignment_search(m.copy())
        fx[f"mas.{name}.durations"] = np.bincount(fx[f"mas.{name}.path"])

    ck, pieces = converter_case()
    state["char_tokenizer"] = _CharTokenizer(pieces)
    ck_in = {k: {n: v.clone() for n, v in d.items()} for k, d in ck.items()}
    out = loader.convert_unity2_aligner_checkpoint(ck_in, cfg)["model"]
    fx["convert.pieces"] = np.array(pieces)
    fx["convert.keys"] = np.array(list(out))
    for k, v in out.items():
        fx[f"convert.out.{k}"] = v.numpy()
    for src, d in ck.items():
        for k, v in d.items():
            fx[f"convert.in.{src}.{k}"] = v.numpy()

    tok = ut.UnitTokenizer(num_units=c["num_units"], langs=c["unit_langs"], model_arch=c["model_arch"])
    front = model.UnitY2AlignmentFrontend(None, None, _CharTokenizer(pieces), tok)
    units = torch.tensor([0, 1, 5, 9999, 10000, 10001, 12345, 3])
    fx["units.in"] = units.numpy()
    fx["units.out"] = front.tokenize_unit(units).numpy()
    fx["units.out_str"] = front.tokenize_unit("7 10003 10004 0").numpy()
    fx["units.vocab_size"] = np.array(tok.vocab_info.size)
    np.savez_compressed(os.path.join(HERE, "aligner.npz"), **fx)
    print("wrote aligner.npz:", len(fx), "arrays")


if __name__ == "__main__":
    main()
