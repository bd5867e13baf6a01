"""Checkpoint ingestion for the S2ST hot path (SURVEY 8f.3): original fairseq-named SeamlessM4T-v2 / vocoder checkpoints
-> the fairseq2 parameter names `UnitYEngine` / `VocoderEngine` consume.

Replaces `convert_unity_checkpoint` + `_fairseq_key_map` (reference: src/seamless_communication/models/unity/loader.py:27-389)
for the model family of this path - w2v-BERT 2.0 Conformer speech encoder with the non-Conformer adaptor, NLLB text
encoder (renamed and kept, not executed by this path) / decoder, NAR T2U (`unity_archs "base_v2"`, the reference's
"X2T/S2T + T2U" branch with a Conformer encoder) - and `convert_vocoder_checkpoint` (models/vocoder/loader.py:20-37).
The Conformer adaptor and the expressive (prosody) variants are outside the path (SURVEY 2) and rejected.  Rules are generated from compact tables;
`tests/test_host_cpu.py` holds them to the mapping produced by the reference's own functions
(tests/golden/make_golden_keymap.py -> unity_keymap.json).

Rename semantics are those of fairseq2's `convert_fairseq_checkpoint` [fs2-recall]: per key, the first rule whose
regex substitution changes the key wins; unmatched keys are kept."""
from __future__ import annotations

import re
from typing import Any, Dict, List, Mapping, Optional, Sequence, Tuple

import torch

_ENC, _DEC, _T2U_ENC, _T2U_DEC = "encoder", "target_letter_decoder", "synthesizer_encoder", "decoder"


def _rules() -> List[Tuple["re.Pattern[str]", str]]:
    L = r"([0-9]+)"
    out: List[Tuple[str, str]] = []

    def add(src_prefix: str, dst_prefix: str, pairs: Sequence[Tuple[str, str]]):
        for a, b in pairs:
            out.append((src_prefix + a, dst_prefix + b))

    w2v = rf"^{_ENC}\.w2v_encoder\.w2v_model\."
    # frontend
    add(w2v, "speech_encoder_frontend.", [
        (r"encoder\.pos_conv\.0\.", "pos_encoder.conv."), (r"layer_norm\.", "post_extract_layer_norm."),
        (r"post_extract_proj\.", "model_dim_proj."),
        (rf"feature_extractor\.conv_layers\.{L}\.0\.", r"feature_extractor.layers.\1.conv."),
        (rf"feature_extractor\.conv_layers\.{L}\.2\.1\.", r"feature_extractor.layers.\1.layer_norm."),
        (r"feature_extractor\.conv_layers\.0\.2\.", "feature_extractor.layers.0.group_norm.")])
    # Conformer blocks (fairseq module name -> fairseq2 module name)
    lay_src, lay_dst = w2v + rf"encoder\.layers\.{L}\.", r"speech_encoder.inner.layers.\1."
    conv = [("batch_norm", "conv.batch_norm"), ("layer_norm2", "conv.layer_norm"), ("depthwise_conv", "conv.depthwise_conv"),
            ("layer_norm", "conv_layer_norm"), ("pointwise_conv1", "conv.pointwise_conv1"), ("pointwise_conv2", "conv.pointwise_conv2")]
    add(lay_src, lay_dst, [(rf"conv_module\.{a}\.", b + ".") for a, b in conv])
    add(lay_src, lay_dst, [(r"ffn(1|2)\.layer_norm\.", r"ffn\2_layer_norm."), (r"ffn(1|2)\.w_1\.", r"ffn\2.inner_proj."),
                           (r"ffn(1|2)\.w_2\.", r"ffn\2.output_proj."), (r"self_attn_layer_norm\.", "self_attn_layer_norm.")])
    attn = [("linear_q", "q_proj"), ("linear_k", "k_proj"), ("linear_v", "v_proj"), ("linear_out", "output_proj"),
            ("q_proj", "q_proj"), ("k_proj", "k_proj"), ("v_proj", "v_proj"), ("rel_k_embedding", "sdpa.rel_k_embed"),
            ("out_proj", "output_proj"), ("linear_pos", "sdpa.r_proj")]
    add(lay_src, lay_dst, [(rf"self_attn\.{a}\.", f"self_attn.{b}.") for a, b in attn])
    add(lay_src, lay_dst, [(r"self_attn\.pos_bias_u", "self_attn.sdpa.u_bias"), (r"self_attn\.pos_bias_v", "self_attn.sdpa.v_bias"),
                           (r"final_layer_norm\.", "layer_norm.")])
    # the stray LayerNorm after the Conformer stack belongs to the adaptor block in fairseq2 (loader.py:266-285)
    add(w2v, "speech_encoder.", [(r"encoder\.layer_norm\.", "inner_layer_norm.")])
    # encoder adaptor
    ad = rf"^{_ENC}\.adaptor\."
    add(ad, "speech_encoder.", [(r"proj\.0\.", "proj1."), (r"proj\.2\.", "proj2."), (r"out_ln\.", "layer_norm.")])
    add(ad + rf"layers\.{L}\.", r"speech_encoder.adaptor_layers.\1.", [
        (r"residual_layer_norm\.", "residual_layer_norm."), (r"residual_pool\.1\.", "residual_conv."), (r"attn_pool\.1\.", "self_attn_conv."),
        (r"self_attn\.out_proj\.", "self_attn.output_proj."), (r"self_attn\.", "self_attn."),
        (r"self_attn_layer_norm\.", "self_attn_layer_norm."), (r"fc1\.", "ffn.inner_proj."), (r"fc2\.", "ffn.output_proj."),
        (r"final_layer_norm\.", "ffn_layer_norm.")])

    def transformer(src: str, dst: str, cross: bool) -> List[Tuple[str, str]]:
        p = [(r"self_attn\.out_proj\.", "self_attn.output_proj."), (r"self_attn\.", "self_attn."),
             (r"self_attn_layer_norm\.", "self_attn_layer_norm.")]
        if cross:
            p += [(r"encoder_attn\.out_proj\.", "encoder_decoder_attn.output_proj."), (r"encoder_attn\.", "encoder_decoder_attn."),
                  (r"encoder_attn_layer_norm\.", "encoder_decoder_attn_layer_norm.")]
        p += [(r"fc1\.", "ffn.inner_proj."), (r"fc2\.", "ffn.output_proj."), (r"final_layer_norm\.", "ffn_layer_norm.")]
        return [(rf"^{src}\.layers\.{L}\." + a, rf"{dst}.layers.\1." + b) for a, b in p]

    # text encoder (part of the multitask checkpoint; renamed for completeness, unused by the S2ST path)
    out.append((r"^text_encoder\.embed_tokens\.", "text_encoder_frontend.embed."))
    out.extend(transformer("text_encoder", "text_encoder", cross=True))
    out.append((r"^text_encoder\.layer_norm\.", "text_encoder.layer_norm."))
    # text decoder
    out.append((rf"^{_DEC}\.embed_tokens\.", "text_decoder_frontend.embed."))
    out.extend(transformer(_DEC, "text_decoder", cross=True))
    out.append((rf"^{_DEC}\.layer_norm\.", "text_decoder.layer_norm."))
    out.append((rf"^{_DEC}\.output_projection\.", "final_proj."))
    # T2U encoder
    out.extend(transformer(_T2U_ENC, "t2u_model.encoder", cross=False))
    out.append((rf"^{_T2U_ENC}\.layer_norm\.", "t2u_model.encoder.layer_norm."))
    # NAR T2U decoder frontend + FFT decoder
    add(rf"^{_T2U_DEC}\.", "t2u_model.decoder_frontend.", [
        (r"embed_tokens_text\.", "embed_char."), (r"embed_tokens_unit\.", "embed."), (r"embed_tokens\.", "embed."),
        (r"var_adaptor\.duration_predictor\.", "variance_adaptor.duration_predictor."), (r"dec_pos_emb_alpha", "pos_emb_alpha"),
        (r"char_upsampler\.pos_emb_alpha", "pos_emb_alpha_char")])
    dl_src, dl_dst = rf"^{_T2U_DEC}\.layers\.{L}\.", r"t2u_model.decoder.layers.\1."
    add(dl_src, dl_dst, [(r"self_attn\.out_proj\.", "self_attn.output_proj."), (r"self_attn\.", "self_attn."),
                         (r"self_attn_layer_norm\.", "self_attn_layer_norm."), (r"layer_norm\.", "self_attn_layer_norm."),
                         (r"encoder_attn\.out_proj\.", "encoder_decoder_attn.output_proj."), (r"encoder_attn\.", "encoder_decoder_attn."),
                         (r"encoder_attn_layer_norm\.", "encoder_decoder_attn_layer_norm."), (r"fc1\.", "ffn.inner_proj."),
                         (r"fc2\.", "ffn.output_proj."), (r"final_layer_norm\.", "ffn_layer_norm."),
                         (r"ffn\.ffn\.0\.", "conv1d.conv1."), (r"ffn\.ffn\.2\.", "conv1d.conv2."), (r"ffn\.layer_norm\.", "conv1d_layer_norm.")])
    out.append((rf"^{_T2U_DEC}\.layer_norm\.", "t2u_model.decoder.layer_norm."))
    out.append((rf"^{_T2U_DEC}\.output_projection\.", "t2u_model.final_proj."))
    return [(re.compile(a), b) for a, b in out]


_RULES: Optional[List[Tuple["re.Pattern[str]", str]]] = None


def rename_key(key: str) -> str:
    """fairseq parameter name -> fairseq2 parameter name (first rule that changes the key wins)."""
    global _RULES
    if _RULES is None:
        _RULES = _rules()
    for pat, rep in _RULES:
        new = pat.sub(rep, key)
        if new != key:
            return new
    return key


def char_index_mapping(char_pieces: Sequence[str]) -> List[int]:
    """Row permutation of the character embedding table: the fairseq dictionary holds the characters in sorted order,
    the SentencePiece model in its own order (loader.py:156-175).  `char_pieces[i]` = piece of index i, incl. the 4
    control symbols."""
    spm_order = list(char_pieces)[4:]
    dict_pos = {ch: idx for idx, ch in zip(range(4, len(char_pieces)), sorted(spm_order))}
    return [0, 1, 2, 3] + [dict_pos[ch] for ch in spm_order]


def convert_unity_checkpoint(checkpoint: Mapping[str, Any], char_pieces: Optional[Sequence[str]] = None,
                             nllb_vocab: int = 256102) -> Dict[str, Any]:
    """{"model": fairseq state dict} -> {"model": fairseq2 state dict}; a checkpoint already in fairseq2 naming passes
    through.  Besides the renames (loader.py:27-153): bookkeeping entries are dropped, NLLB-100's dummy last embedding
    row is discarded, the tied embedding tables are unified, the control-symbol rows are permuted
    (BOS, PAD, EOS, UNK) -> (PAD, UNK, BOS, EOS), and the character embeddings are permuted to the SentencePiece order
    (needs `char_pieces`)."""
    sd = checkpoint["model"]
    if "speech_encoder.inner.layers.0.self_attn_layer_norm.weight" in sd:
        return dict(checkpoint)
    if any(k.startswith(("s2t_model.", "t2s_model.")) for k in sd):
        raise NotImplementedError("expressive (prosody) checkpoints are outside the S2ST hot path (SURVEY 2)")
    has_text_encoder = any(k.startswith("text_encoder.") for k in sd)
    out = {rename_key(k): v for k, v in sd.items()}
    # fairseq2's generic converter drops these on its own [fs2-recall]; harmless if absent
    for k in ("encoder.version", "decoder.version", "encoder.embed_positions._float_tensor", "decoder.embed_positions._float_tensor"):
        out.pop(k, None)
    drop = ["text_encoder.version", "text_encoder.embed_positions._float_tensor",
            f"{_DEC}.version", f"{_DEC}.embed_positions._float_tensor", f"{_ENC}.w2v_encoder.w2v_model.mask_emb",
            f"{_T2U_DEC}.char_upsampler.embed_positions._float_tensor", f"{_T2U_DEC}.char_upsampler.embed_tokens_char.weight",
            "decoder_target_letter_decoder.proj.weight", "decoder_target_letter_decoder.proj.bias"]
    drop += [k for k in out if k.startswith(f"{_T2U_DEC}.alignment_encoder.")]
    for k in drop:
        out.pop(k, None)
    embeds = out["final_proj.weight"]
    if embeds.size(0) == nllb_vocab + 1:  # fairseq's accidental dummy token at the end of NLLB-100's table
        embeds = embeds[:-1]
        out["final_proj.weight"] = embeds
    out["text_decoder_frontend.embed.weight"] = embeds  # one tied table
    if has_text_encoder:
        out["text_encoder_frontend.embed.weight"] = embeds
    with torch.inference_mode():
        embeds[[0, 1, 2, 3]] = embeds[[1, 3, 0, 2]]
    ce = out.get("t2u_model.decoder_frontend.embed_char.weight")
    if ce is not None:
        if char_pieces is None:
            raise ValueError("char_pieces (the character SentencePiece vocabulary) is needed to permute embed_char")
        idx = char_index_mapping(char_pieces)
        with torch.inference_mode():
            ce[torch.arange(len(idx))] = ce[idx]
    if "t2u_model.final_proj.weight" in out and "t2u_model.decoder_frontend.embed.weight" in out:
        out["t2u_model.decoder_frontend.embed.weight"] = out["t2u_model.final_proj.weight"]
    return {"model": out}


def convert_vocoder_checkpoint(checkpoint: Mapping[str, Any]) -> Dict[str, Any]:
    """{"generator": hifigan state dict} -> {"model": {"code_generator.<key>": ...}} (vocoder/loader.py:20-37)."""
    if "model" in checkpoint and "code_generator.resblocks.0.convs1.0.weight_g" in checkpoint["model"]:
        return dict(checkpoint)
    out = {k: v for k, v in checkpoint.items() if k != "generator"}
    out["model"] = {f"code_generator.{k}": v for k, v in checkpoint["generator"].items()}
    return out


_W2V2_RULES = [(re.compile(a), b) for a, b in (
    # frontend, as the reference's conformer_shaw/loader.py:44-70 maps a fairseq wav2vec2 model
    (r"^encoder\.pos_conv\.0\.", "encoder_frontend.pos_encoder.conv."),
    (r"^feature_extractor\.conv_layers\.([0-9]+)\.0\.", r"encoder_frontend.feature_extractor.layers.\1.conv."),
    (r"^feature_extractor\.conv_layers\.([0-9]+)\.2\.1\.", r"encoder_frontend.feature_extractor.layers.\1.layer_norm."),
    (r"^layer_norm\.", "encoder_frontend.post_extract_layer_norm."),
    (r"^post_extract_proj\.", "encoder_frontend.model_dim_proj."),
    # plain pre-LN Transformer layers (fairseq2's wav2vec2 loader; recalled, DESIGN.md section 11)
    (r"^encoder\.layers\.([0-9]+)\.self_attn\.out_proj\.", r"encoder.layers.\1.self_attn.output_proj."),
    (r"^encoder\.layers\.([0-9]+)\.fc1\.", r"encoder.layers.\1.ffn.inner_proj."),
    (r"^encoder\.layers\.([0-9]+)\.fc2\.", r"encoder.layers.\1.ffn.output_proj."),
    (r"^encoder\.layers\.([0-9]+)\.final_layer_norm\.", r"encoder.layers.\1.ffn_layer_norm."),
)]


def convert_wav2vec2_checkpoint(checkpoint: Mapping[str, Any]) -> Dict[str, Any]:
    """fairseq `xlsr2_1b_v2.pt` ({"model": fairseq names}) -> {"model": fairseq2 names}.  Keys no rule matches keep their
    name (self_attn.{q,k,v}_proj, self_attn_layer_norm and encoder.layer_norm are spelled alike in both); a dict already
    in fairseq2 names passes through unchanged."""
    sd = checkpoint.get("model", checkpoint)
    if any(k.startswith("encoder_frontend.") for k in sd):
        return {"model": dict(sd)}
    out: Dict[str, Any] = {}
    for k, v in sd.items():
        for pat, rep in _W2V2_RULES:
            if pat.search(k):
                k = pat.sub(rep, k)
                break
        out[k] = v
    return {"model": out}


def convert_unity2_aligner_checkpoint(checkpoint: Mapping[str, Any], char_pieces: Sequence[str]) -> Dict[str, Any]:
    """UnitY2 aligner checkpoint (`unity2_aligner.pt`: text_emb_state / unit_emb_state / aligner_state) -> {"model": names of
    UnitY2AlignmentModel} (reference models/aligner/loader.py:22-74); one that already holds
    `model["alignment_encoder.t_conv.1.weight"]` passes through.  The character embedding rows are permuted from the
    fairseq dictionary's sorted order to the SentencePiece order (`char_index_mapping(char_pieces)`) on a copy: the input
    tensors are left as they are (the reference permutes them in place)."""
    if "model" in checkpoint and "alignment_encoder.t_conv.1.weight" in checkpoint["model"]:
        return dict(checkpoint)
    model: Dict[str, Any] = {f"alignment_encoder.{k}": v for k, v in checkpoint["aligner_state"].items()}
    for src, name in (("text_emb_state", "embed_text"), ("unit_emb_state", "embed_unit")):
        for k, v in checkpoint[src].items():
            if k != "weight":
                raise KeyError(f"unexpected key '{k}' in {src}")
            model[f"alignment_frontend.{name}.weight"] = v
    idx = char_index_mapping(char_pieces)
    ce = model["alignment_frontend.embed_text.weight"].clone()
    with torch.inference_mode():
        ce[torch.arange(len(idx))] = ce[idx]
    model["alignment_frontend.embed_text.weight"] = ce
    return {**checkpoint, "model": model}


def load_checkpoint_file(path: str) -> Dict[str, Any]:
    return torch.load(path, map_location="cpu", weights_only=True)
