"""Architecture configuration for the S2ST hot path.

Mirrors the hyper-parameters the reference keeps in its architecture
registries (reference: src/seamless_communication/models/unity/builder.py:165-192
`_base_v2`, models/unity/t2u_builder.py:186-232 `_base_nar`,
models/conformer_shaw/builder.py:55-68, models/vocoder/builder.py:42-64
`_base_vocoder`).  Only the fields the hot path reads are kept.

Named architectures:
  * ``base_v2``  - seamlessM4T_v2_large (the headline configuration);
  * ``tiny_v2`` / ``small_v2`` - same topology, small dims / few layers, used by
    the parity tests so the CPU oracle finishes in seconds;
  * ``base``     - seamlessM4T_large (builder.py:109-134, w2v-BERT v1 speech
    encoder, same 600m / dense_1b dims), with ``tiny_v1`` / ``small_v1`` test
    copies.  Their T2U is the autoregressive one (t2u_builder.py:141-160
    `_base_t2u`): a pre-LN Transformer encoder and an NLLB-type decoder over the
    unit vocabulary, sized by the same ``t2u_*`` / ``unit_*`` fields.
"""
from __future__ import annotations

from dataclasses import dataclass, field, asdict
from typing import Dict, List, Tuple

# Languages of the reference asset cards (cards/unity_nllb-100.yaml `langs`,
# cards/seamlessM4T_v2_large.yaml `unit_langs`, cards/vocoder_v2.yaml).  These
# are configuration data the API surface exposes (tgt_lang validation).
NLLB100_LANGS: Tuple[str, ...] = tuple(
    "afr amh arb ary arz asm azj bel ben bos bul cat ceb ces ckb cmn cmn_Hant cym dan deu ell eng est eus "
    "fin fra fuv gaz gle glg guj heb hin hrv hun hye ibo ind isl ita jav jpn kan kat kaz khk khm kir kor lao "
    "lit lug luo lvs mai mal mar mkd mlt mni mya nld nno nob npi nya ory pan pbt pes pol por ron rus sat slk "
    "slv sna snd som spa srp swe swh tam tel tgk tgl tha tur ukr urd uzn vie yor yue zsm zul".split()
)
UNIT_LANGS_V2: Tuple[str, ...] = tuple(
    "arb ben cat ces cmn cym dan deu eng est fin fra hin ind ita jpn kan kor mlt nld pes pol por ron rus slk "
    "spa swe swh tam tel tgl tha tur ukr urd uzn vie".split()
)
VOCODER_LANGS_V2: Tuple[str, ...] = tuple(
    "arb ben cat ces cmn cym dan deu eng est fin fra hin ind ita jpn kor mlt nld pes pol por ron rus slk spa "
    "swe swh tel tgl tha tur ukr urd uzn vie".split()
)
# first speaker id per language (cards/vocoder_v2.yaml model_config.lang_spkr_idx_map.multispkr)
_VOCODER_SPKR_COUNTS = [1, 1, 1, 1, 2, 1, 2, 1, 1, 3, 1, 1, 1, 11, 2, 1, 1, 3, 3, 1, 1, 1, 1, 2, 1, 1, 3, 3, 1, 1,
                        5, 3, 1, 3, 3, 6]
# the card lists speaker ids per language; only the *first* is ever used by the
# path (vocoder.py:44).  First ids as in the card:
_VOCODER_FIRST_SPKR = [0, 1, 2, 3, 4, 6, 7, 9, 10, 11, 14, 15, 16, 17, 29, 30, 31, 32, 35, 38, 39, 40, 41, 43,
                       44, 45, 46, 49, 52, 53, 54, 61, 62, 63, 66, 69]


# first speaker id per language of cards/vocoder_36langs.yaml (seamlessM4T_large's vocoder; same 36 languages in the
# same order, different speaker table: tests/golden/vocoder_36langs_map.json holds the card's whole map)
_VOCODER36_FIRST_SPKR = [0, 2, 3, 4, 5, 6, 7, 9, 10, 11, 14, 15, 16, 17, 29, 30, 31, 32, 35, 36, 37, 38, 39, 40, 41,
                         42, 43, 46, 49, 50, 51, 58, 59, 60, 63, 66]


def vocoder_lang_spkr_idx_map(card: str = "vocoder_v2") -> Dict[str, Dict]:
    first = _VOCODER36_FIRST_SPKR if card == "vocoder_36langs" else _VOCODER_FIRST_SPKR
    return {
        "multilingual": {l: i for i, l in enumerate(VOCODER_LANGS_V2)},
        "multispkr": {l: [first[i]] for i, l in enumerate(VOCODER_LANGS_V2)},
    }


@dataclass
class UnitYConfig:
    """Flat config of the whole S2ST stack (speech encoder, text decoder, T2U).  The T2U is non-autoregressive for
    encoder_variant "v2" and autoregressive for "v1" (seamlessM4T_large)."""

    name: str = "base_v2"
    model_dim: int = 1024
    num_heads: int = 16  # head_dim is fixed at 64 by the attention kernels
    # --- w2v-BERT 2.0 conformer (conformer_shaw "600m") ---
    fbank_channels: int = 80
    fbank_stride: int = 2
    enc_layers: int = 24
    enc_ffn_dim: int = 4096
    dw_kernel: int = 31
    shaw_left: int = 64
    shaw_right: int = 8
    # "v2": Shaw relative attention, causal depthwise conv + LayerNorm (w2v-BERT 2.0);
    # "v1": Transformer-XL relative attention, symmetric depthwise conv + BatchNorm (w2v-BERT v1, seamlessM4T_large)
    encoder_variant: str = "v2"
    # --- adaptor (builder.py:188-192) ---
    adaptor_kernel: int = 8
    adaptor_stride: int = 8
    # --- NLLB text decoder (nllb "dense_1b") ---
    dec_layers: int = 24
    dec_ffn_dim: int = 8192
    text_vocab: int = 256102
    text_pad: int = 0
    text_unk: int = 1
    text_bos: int = 2
    text_eos: int = 3
    # --- T2U: NAR "base_nar" (v2) or AR "base" (v1, t2u_builder.py:141-160); both 6 + 6 layers, FFN 8192 ---
    t2u_enc_layers: int = 6
    t2u_dec_layers: int = 6
    t2u_ffn_dim: int = 8192
    unit_vocab: int = 10082  # AR: num_units + 2 * (len(unit_langs) + 1) + 4
    num_units: int = 10000
    unit_pad: int = 1
    unit_eos: int = 2
    unit_bos: int = 0
    unit_unk: int = 3
    unit_max_seq_len: int = 2048  # position table of the AR T2U decoder
    char_vocab: int = 10943
    char_pad: int = 1
    fft_kernel: int = 7
    fft_inner_dim: int = 1024
    var_hidden: int = 256
    var_kernel: int = 3
    max_seq_len: int = 4096
    langs: Tuple[str, ...] = NLLB100_LANGS
    unit_langs: Tuple[str, ...] = UNIT_LANGS_V2

    @property
    def head_dim(self) -> int:
        return self.model_dim // self.num_heads

    def to_dict(self) -> Dict:
        return asdict(self)


@dataclass
class VocoderConfig:
    """vocoder_code_hifigan "base" (models/vocoder/builder.py:42-64)."""

    name: str = "base"
    upsample_rates: Tuple[int, ...] = (5, 4, 4, 2, 2)
    upsample_kernel_sizes: Tuple[int, ...] = (11, 8, 8, 4, 4)
    upsample_initial_channel: int = 512
    resblock_kernel_sizes: Tuple[int, ...] = (3, 7, 11)
    resblock_dilation_sizes: Tuple[Tuple[int, ...], ...] = ((1, 3, 5), (1, 3, 5), (1, 3, 5))
    num_embeddings: int = 10000
    embedding_dim: int = 1280
    lang_embedding_dim: int = 256
    num_langs: int = 36
    spkr_embedding_dim: int = 256
    num_spkrs: int = 200
    # duration predictor (dur_predictor_params of builder.py:53-58): VariancePredictor over the unit embeddings
    var_pred_hidden: int = 1280
    var_pred_kernel: int = 3
    langs: Tuple[str, ...] = VOCODER_LANGS_V2

    @property
    def model_in_dim(self) -> int:
        return self.embedding_dim + self.lang_embedding_dim + self.spkr_embedding_dim

    @property
    def hop(self) -> int:
        h = 1
        for u in self.upsample_rates:
            h *= u
        return h

    def to_dict(self) -> Dict:
        return asdict(self)


def base_v2() -> UnitYConfig:
    return UnitYConfig()


def tiny_v2() -> UnitYConfig:
    """Same topology as base_v2, dims shrunk so the fp32 CPU oracle runs in seconds."""
    return UnitYConfig(
        name="tiny_v2",
        model_dim=128,
        num_heads=2,
        enc_layers=2,
        enc_ffn_dim=256,
        dec_layers=2,
        dec_ffn_dim=256,
        text_vocab=1024 + 102,
        t2u_enc_layers=1,
        t2u_dec_layers=2,
        t2u_ffn_dim=256,
        unit_vocab=256 + 82,
        num_units=256,
        char_vocab=64,
        fft_inner_dim=128,
        var_hidden=64,
        max_seq_len=2048,
    )


def small_v2() -> UnitYConfig:
    """Mid-size: full widths (1024, 16 heads) but few layers / small vocab; GPU parity at real tile shapes."""
    return UnitYConfig(
        name="small_v2",
        enc_layers=2,
        dec_layers=2,
        text_vocab=8192 + 102,
        t2u_enc_layers=1,
        t2u_dec_layers=1,
        max_seq_len=1024,
    )


def base() -> UnitYConfig:
    """seamlessM4T_large: the base_v2 dims with the w2v-BERT v1 encoder and the autoregressive T2U."""
    return UnitYConfig(name="base", encoder_variant="v1")


def tiny_v1() -> UnitYConfig:
    c = tiny_v2()
    c.name, c.encoder_variant = "tiny_v1", "v1"
    return c


def small_v1() -> UnitYConfig:
    c = small_v2()
    c.name, c.encoder_variant = "small_v1", "v1"
    return c


def base_vocoder() -> VocoderConfig:
    return VocoderConfig()


def tiny_vocoder() -> VocoderConfig:
    return VocoderConfig(
        name="tiny",
        upsample_initial_channel=256,
        num_embeddings=256,
        embedding_dim=64,
        lang_embedding_dim=32,
        spkr_embedding_dim=32,
        var_pred_hidden=64,
    )


UNITY_ARCHS = {"base_v2": base_v2, "tiny_v2": tiny_v2, "small_v2": small_v2, "base": base, "tiny_v1": tiny_v1,
               "small_v1": small_v1}
VOCODER_ARCHS = {"base": base_vocoder, "tiny": tiny_vocoder}

# asset-card names the reference resolves through fairseq2's asset store
# (cards/seamlessM4T_v2_large.yaml: model_arch base_v2; cards/vocoder_v2.yaml and vocoder_36langs.yaml: base)
MODEL_CARDS = {"seamlessM4T_v2_large": "base_v2", "seamlessM4T_v2_tiny": "tiny_v2", "seamlessM4T_v2_small": "small_v2",
               "seamlessM4T_large": "base"}
VOCODER_CARDS = {"vocoder_v2": "base", "vocoder_v2_tiny": "tiny", "vocoder_36langs": "base"}
