#!/usr/bin/env python
"""Generates tests/golden/unit_extractor.json by EXECUTING the reference's own code here (needs the reference tree;
nothing is copied):

  * `_encoder_xlsr2_1b_v2` / `_xlsr2_1b_v2` (models/unit_extractor/wav2vec2_layer_output.py:23-75), run with dataclass
    stand-ins for fairseq2's Wav2Vec2EncoderConfig / Wav2Vec2Config that accept and record every field, so the fixture
    pins every field of the architecture;
  * `KmeansModel` (models/unit_extractor/kmeans.py), loaded from a seeded `.npy` through a download-manager stand-in and
    run on seeded features; the centroids contain exact duplicates (a tie goes to the lowest index) and K = 300 is not a
    multiple of 128;
  * the fairseq -> fairseq2 key map of conformer_shaw/loader.py:44-70 (taken out of the source with `ast`), applied to
    one example key per frontend rule.

and writes tests/golden/w2v2_encoder_ref.npz from the reference's C++ mirror of fairseq2 (`ggml/examples/unity/
fairseq2.cpp`, compiled into oracle/_ref/libfairseq2_ref.so by `oracle/Makefile`): `fs2ref_encoder`, i.e.
StandardTransformerEncoder_forward (fairseq2.cpp:502-552, 955-977: pre-LN layers with a ReLU FFN, then the final
LayerNorm), at head_dim 80 (160 wide, 2 heads, 2 layers) on unpadded sequences, called as make_golden_beam.py calls it.
The weights come from `mirror_encoder_state_dict(seed)`, which the test regenerates; the fixture stores x and y.
"""
import ast
import enum
import importlib.util
import json
import os
import re
import sys
import tempfile
import types

import numpy as np
import torch

REF = "/root/reference/src/seamless_communication/models"
HERE = os.path.dirname(os.path.abspath(__file__))
MIRROR = {"model_dim": 160, "num_heads": 2, "ffn_dim": 320, "layers": 2, "prefix": "encoder"}
MIRROR_CASES = ((1, 37), (2, 1), (3, 70))  # (seed, sequence length)


def mirror_encoder_state_dict(seed: int):
    """fp32 pre-LN encoder weights under fairseq2's names (prefix "encoder"), head_dim 80."""
    M, Fd = MIRROR["model_dim"], MIRROR["ffn_dim"]
    g = torch.Generator().manual_seed(5000 + seed)
    sd = {}

    def lin(p, o, i):
        sd[p + ".weight"] = torch.randn(o, i, generator=g) * (2.0 / (o + i)) ** 0.5 * 1.5
        sd[p + ".bias"] = torch.randn(o, generator=g) * 0.05

    def ln(p):
        sd[p + ".weight"] = 1.0 + 0.1 * torch.randn(M, generator=g)
        sd[p + ".bias"] = 0.05 * torch.randn(M, generator=g)

    for i in range(MIRROR["layers"]):
        p = f"{MIRROR['prefix']}.layers.{i}"
        ln(p + ".self_attn_layer_norm")
        for q in ("q_proj", "k_proj", "v_proj", "output_proj"):
            lin(f"{p}.self_attn.{q}", M, M)
        ln(p + ".ffn_layer_norm")
        lin(p + ".ffn.inner_proj", Fd, M)
        lin(p + ".ffn.output_proj", M, Fd)
    ln(MIRROR["prefix"] + ".layer_norm")
    return sd


def mirror_input(seed: int, S: int):
    return torch.randn(S, MIRROR["model_dim"], generator=torch.Generator().manual_seed(6000 + seed))


class _Config:
    """Accepts any keyword (or positional) fields and keeps them in order."""

    def __init__(self, *args, **kw):
        self.args, self.fields = list(args), dict(kw)


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class TransformerNormOrder(enum.Enum):
    POST = 0
    PRE = 1
    PRE_WITH_NORMFORMER = 2


def _jsonable(v):
    if isinstance(v, enum.Enum):
        return v.name
    if isinstance(v, (list, tuple)):
        return [_jsonable(x) for x in v]
    return v


def arch_fields():
    archs = {}
    _stub("fairseq2")
    _stub("fairseq2.models")
    _stub("fairseq2.models.sequence", SequenceBatch=object)
    _stub("fairseq2.models.wav2vec2", Wav2Vec2Config=_Config, Wav2Vec2EncoderConfig=_Config, Wav2Vec2Frontend=object,
          Wav2Vec2Model=object, wav2vec2_arch=lambda name: (lambda f: archs.setdefault(name, f)))
    _stub("fairseq2.nn")
    _stub("fairseq2.nn.padding", PaddingMask=object)
    _stub("fairseq2.nn.transformer", TransformerEncoder=object, TransformerNormOrder=TransformerNormOrder)
    spec = importlib.util.spec_from_file_location("w2v2_layer_output", os.path.join(REF, "unit_extractor", "wav2vec2_layer_output.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    enc = mod._encoder_xlsr2_1b_v2()
    full = archs["xlsr2_1b_v2"]()
    return {"encoder": {k: _jsonable(v) for k, v in enc.fields.items()},
            "model": {k: _jsonable(v) for k, v in full.fields.items()}}


def kmeans_case():
    g = torch.Generator().manual_seed(11)
    K, D, N = 300, 64, 96
    c = torch.randn(K, D, generator=g)
    c[200] = c[7]     # exact duplicates: frames nearest to them must get index 7 / 50
    c[299] = c[50]
    x = torch.randn(N, D, generator=g)
    x[:8] = c[7] + 0.01 * torch.randn(8, D, generator=g)
    x[8:16] = c[50] + 0.01 * torch.randn(8, D, generator=g)
    x[16] = c[299]
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "km.npy")
        np.save(path, c.numpy())  # the file holds (K, D); KmeansModel transposes it to (D, K)
        _stub("fairseq2.assets", download_manager=types.SimpleNamespace(download_checkpoint=lambda uri, name: uri))
        _stub("fairseq2.typing", DataType=object, Device=object)
        spec = importlib.util.spec_from_file_location("kmeans_ref", os.path.join(REF, "unit_extractor", "kmeans.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        units = mod.KmeansModel(path, torch.device("cpu"), torch.float32)(x)
    return {"seed": 11, "K": K, "D": D, "N": N, "units": units.tolist()}


def frontend_keys():
    src = open(os.path.join(REF, "conformer_shaw", "loader.py")).read()
    tree = ast.parse(src)
    key_map = None
    for node in ast.walk(tree):
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "key_map" for t in node.targets):
            key_map = ast.literal_eval(node.value)
    assert key_map is not None
    examples = ["encoder.pos_conv.0.weight_g", "encoder.pos_conv.0.weight_v", "encoder.pos_conv.0.bias",
                "feature_extractor.conv_layers.3.0.weight", "feature_extractor.conv_layers.0.0.bias",
                "feature_extractor.conv_layers.5.2.1.weight", "layer_norm.bias", "post_extract_proj.weight",
                "encoder.layers.12.self_attn.out_proj.weight", "encoder.layers.3.fc1.bias", "encoder.layers.47.fc2.weight"]
    out = {}
    for k in examples:
        for pat, rep in key_map.items():  # fairseq2's convert_fairseq_checkpoint: the first rule that changes the key wins
            n = re.sub(pat, rep, k)
            if n != k:
                k_new = n
                break
        else:
            k_new = k
        out[k] = k_new
    return out


def mirror_encoder_cases():
    import ctypes as C
    lib = C.CDLL(os.path.join(HERE, "..", "..", "oracle", "_ref", "libfairseq2_ref.so"))
    I, D, PP = C.c_int, C.c_double, C.c_void_p
    lib.fs2ref_encoder.restype = I
    lib.fs2ref_encoder.argtypes = [I, PP, PP, PP, PP, I, PP, I, PP, D, I, PP, I, I, PP, C.c_char_p, PP, I, I, PP]
    P = MIRROR["prefix"]
    cases = {}
    for seed, S in MIRROR_CASES:
        sd = mirror_encoder_state_dict(seed)
        names = sorted(sd)
        arrs = [np.ascontiguousarray(sd[k].numpy().astype(np.float32)) for k in names]
        n = len(names)
        c_names = (C.c_char_p * n)(*[k.encode() for k in names])
        c_data = (C.c_void_p * n)(*[a.ctypes.data for a in arrs])
        d0 = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
        d1 = (C.c_int64 * n)(*[a.shape[1] if a.ndim == 2 else 0 for a in arrs])
        layers = [f"{P}.layers.{i}" for i in range(MIRROR["layers"])]
        attn = [l + ".self_attn" for l in layers]
        lns = [f"{l}.{a}" for l in layers for a in ("self_attn_layer_norm", "ffn_layer_norm")] + [P + ".layer_norm"]
        modules = layers + attn + lns + [l + ".ffn" for l in layers]
        keep = [(C.c_char_p * len(xs))(*[x.encode() for x in xs]) for xs in (modules, lns, attn, layers)]
        x = mirror_input(seed, S).numpy().astype(np.float32)
        y = np.zeros_like(x)
        rc = lib.fs2ref_encoder(n, C.cast(c_names, PP), C.cast(c_data, PP), C.cast(d0, PP), C.cast(d1, PP), len(modules),
                                C.cast(keep[0], PP), len(lns), C.cast(keep[1], PP), 1e-5, len(attn), C.cast(keep[2], PP),
                                MIRROR["num_heads"], len(layers), C.cast(keep[3], PP), P.encode(), x.ctypes.data, S,
                                MIRROR["model_dim"], y.ctypes.data)
        assert rc == 0
        cases[f"x_{seed}"], cases[f"y_{seed}"] = x, y
    return cases


if __name__ == "__main__":
    fx = {"arch": arch_fields(), "kmeans": kmeans_case(), "frontend_keys": frontend_keys()}
    with open(os.path.join(HERE, "unit_extractor.json"), "w") as f:
        json.dump(fx, f, indent=1, sort_keys=True)
    print("wrote unit_extractor.json")
    cases = mirror_encoder_cases()
    np.savez_compressed(os.path.join(HERE, "w2v2_encoder_ref.npz"), **cases)
    print("wrote w2v2_encoder_ref.npz", {k: v.shape for k, v in cases.items()})
