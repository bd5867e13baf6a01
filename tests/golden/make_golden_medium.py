#!/usr/bin/env python
"""Generates tests/golden/medium_card.json: what the reference states about seamlessM4T_medium.

  * `_medium` and `_base` of src/seamless_communication/models/unity/builder.py, read with `ast`: the w2v-BERT and
    NLLB architecture names, the vocabulary size assigned to `mt_model_config.vocab_info.size`, and the keywords of
    the UnitYConfig they return (adaptor included);
  * `_medium_t2u` and `_base_t2u` of models/unity/t2u_builder.py: the keywords of the UnitYT2UConfig, with
    `target_vocab_info` as its keywords;
  * cards/seamlessM4T_medium.yaml, cards/seamlessM4T_large.yaml, cards/unity_nllb-200.yaml: name, base card,
    architecture, num_units, unit_langs and langs, in card order;
  * docs/m4t/README.md: the line that names the vocoder of seamlessM4T_medium.

Run from the repo root (needs /root/reference and PyYAML; the tests only read the committed fixture):

    python tests/golden/make_golden_medium.py
"""
import ast
import json
import os

import yaml

REF = "/root/reference"
SRC = os.path.join(REF, "src/seamless_communication")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "medium_card.json")


def _literal(node):
    """Python value of a constant, a `1024 * 8` product, or a call's keywords (as a dict)."""
    if isinstance(node, ast.Call):
        return {kw.arg: _literal(kw.value) for kw in node.keywords}
    if isinstance(node, ast.BinOp) and isinstance(node.op, ast.Mult):
        return _literal(node.left) * _literal(node.right)
    if isinstance(node, ast.Name):
        return {"None": None, "True": True, "False": False}.get(node.id, f"<name {node.id}>")
    if isinstance(node, ast.Attribute):
        return f"<attr {ast.unparse(node)}>"
    return ast.literal_eval(node)


def _functions(path):
    return {f.name: f for f in ast.parse(open(path).read()).body if isinstance(f, ast.FunctionDef)}


def _builder(fn):
    out = {"archs": {}}
    for node in ast.walk(fn):
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "get_config":
            out["archs"][ast.unparse(node.func.value)] = ast.literal_eval(node.args[0])
        if isinstance(node, ast.Assign) and ast.unparse(node.targets[0]) == "mt_model_config.vocab_info.size":
            out["text_vocab"] = ast.literal_eval(node.value)
        if isinstance(node, ast.Return):
            out["config"] = _literal(node.value)
    return out


def _t2u(fn):
    ret = next(n for n in ast.walk(fn) if isinstance(n, ast.Return))
    return _literal(ret.value)


def _card(name):
    d = yaml.safe_load(open(os.path.join(SRC, "cards", name + ".yaml")))
    return {k: d[k] for k in ("name", "base", "model_arch", "num_units", "unit_langs", "langs", "model_type") if k in d}


def main():
    b = _functions(os.path.join(SRC, "models/unity/builder.py"))
    t = _functions(os.path.join(SRC, "models/unity/t2u_builder.py"))
    readme = [line.strip() for line in open(os.path.join(REF, "docs/m4t/README.md")) if "vocoder_36langs" in line and "medium" in line]
    out = {"builder": {"medium": _builder(b["_medium"]), "base": _builder(b["_base"])},
           "t2u_builder": {"medium": _t2u(t["_medium_t2u"]), "base": _t2u(t["_base_t2u"])},
           "cards": {n: _card(n) for n in ("seamlessM4T_medium", "seamlessM4T_large", "unity_nllb-200", "unity_nllb-100")},
           "readme_vocoder_lines": readme}
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
