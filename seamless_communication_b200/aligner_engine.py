"""Host-side orchestration of the UnitY2 forced aligner (DESIGN.md section 12) on the C-ABI kernels.

`AlignerEngine` packs a `nar_t2u_aligner` state dict (reference names, models/checkpoint.py
`convert_unity2_aligner_checkpoint`) once and runs a ragged batch of (characters, units) rows through
  sb_vocoder_embed (a plain table gather) -> text convs / feature convs on sb_gemm -> sb_align_lprob -> sb_monotonic_align.

Layouts.  Each branch runs in a sequence layout with one zero halo row on both sides of every row and the valid lengths
as the GEMM's row mask, so a k3 conv (3 taps from a_row0 = -1) sees zeros before a row and past its length: row b is
computed as that row alone, which is what the reference's batch-1 `UnitY2AlignmentModel.forward` does (its batched encoder
would let a padded neighbour into the k3 conv).  Padded positions gather an all-zero row appended to each packed table.
The last conv of each branch (k1, a Linear) writes fp32, which sb_align_lprob reads.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import _lib, ops
from .config import AlignerConfig
from .ops import ACT_RELU, F16, Seq

I32 = torch.int32
GEMM_MAX_ROW_TILES = 65535  # sb_gemm puts the 128-row tiles of M on gridDim.y
MAX_TEXT = 8192  # sb_monotonic_align keeps a row's Q column in shared memory


def _as_list(x: Union[torch.Tensor, Sequence[int]]) -> List[int]:
    return [int(v) for v in (x.tolist() if isinstance(x, torch.Tensor) else x)]


class AlignerEngine:
    def __init__(self, cfg: AlignerConfig, state_dict: Dict[str, torch.Tensor], device="cuda"):
        if cfg.reduction_factor != 1:
            raise ValueError(f"reduction_factor {cfg.reduction_factor} is not supported; every aligner card uses 1")
        _lib.require_cuda()
        self.cfg = cfg
        self.device = torch.device(device)
        self._pack(state_dict)

    def _pack(self, sd):
        dev, cfg = self.device, self.cfg

        def table(name, rows, width):
            t = sd[name]
            if tuple(t.shape) != (rows, width):
                raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {(rows, width)}")
            return torch.cat([t.to(F16), torch.zeros(1, width, dtype=F16)]).to(dev).contiguous()  # last row: padding

        def convs(prefix, n, c_in):
            out = []
            for i in range(n):
                k = 3 if i < n - 1 else 1
                w = sd[f"{prefix}.{1 + 3 * i}.weight"]
                if tuple(w.shape) != (cfg.model_dim, c_in, k):
                    raise ValueError(f"{prefix}.{1 + 3 * i}.weight has shape {tuple(w.shape)}, expected {(cfg.model_dim, c_in, k)}")
                # Conv1d (out, in, k) -> sb_gemm's (out, k * in)
                out.append((w.permute(0, 2, 1).reshape(cfg.model_dim, k * c_in).to(dev, F16).contiguous(),
                            sd[f"{prefix}.{1 + 3 * i}.bias"].to(dev, torch.float32).contiguous(), k))
                c_in = cfg.model_dim
            return out

        self.embed_text = table("alignment_frontend.embed_text.weight", cfg.text_vocab_size, cfg.model_dim)
        self.embed_unit = table("alignment_frontend.embed_unit.weight", cfg.unit_vocab_size, cfg.feat_dim)
        self.t_conv = convs("alignment_encoder.t_conv", cfg.num_text_layers, cfg.model_dim)
        self.f_conv = convs("alignment_encoder.f_conv", cfg.num_feat_layers, cfg.feat_dim)

    def _ids(self, ids: torch.Tensor, lens: List[int], vocab: int, what: str) -> torch.Tensor:
        """(B, T) ids -> int32 on the device with every position past a row's length pointing at the zero row."""
        ids = torch.as_tensor(ids).to("cpu", torch.int64)
        if ids.dim() != 2 or ids.shape[0] != len(lens):
            raise ValueError(f"{what} ids must be (B, T) with one length per row; got {tuple(ids.shape)} and {len(lens)} lengths")
        if min(lens) <= 0:
            raise ValueError(f"every row needs at least one {what} position (lengths {lens})")
        if max(lens) > ids.shape[1]:
            raise ValueError(f"a {what} length of {max(lens)} exceeds the id matrix's {ids.shape[1]} columns")
        T = max(lens)
        out = torch.full((len(lens), T), vocab, dtype=torch.int64)
        for b, n in enumerate(lens):
            row = ids[b, :n]
            if n and (int(row.min()) < 0 or int(row.max()) >= vocab):
                raise IndexError(f"{what} id out of range for the {vocab}-entry table (min {int(row.min())}, max {int(row.max())})")
            out[b, :n] = row
        return out.to(self.device, I32)

    def _embed(self, ids: torch.Tensor, lens: torch.Tensor, table: torch.Tensor) -> Seq:
        B, T = ids.shape
        C = table.shape[1]
        x = Seq(B, T, C, halo=1, lens=lens, device=self.device, zero=True)
        zero_idx = torch.zeros(B, dtype=I32, device=self.device)
        lib = _lib.load()
        p = table.data_ptr()
        _lib.check(lib.sb_vocoder_embed(ids.data_ptr(), T, B, p, C, p, 0, zero_idx.data_ptr(), p, 0, zero_idx.data_ptr(),
                                        x.buf.data_ptr(), x.Tp, x.PH, ops._stream()), "sb_vocoder_embed")
        return x

    @staticmethod
    def _convs(x: Seq, layers) -> Seq:
        for i, (w, b, k) in enumerate(layers):
            last = i == len(layers) - 1
            x = ops.gemm(x, w, w.shape[0], b, taps=k, act=0 if last else ACT_RELU, out_f32=last)
        return x

    def check_batch(self, text_lens: List[int], unit_lens: List[int]) -> None:
        if len(text_lens) == 0 or len(text_lens) != len(unit_lens):
            raise ValueError(f"{len(text_lens)} text lengths for {len(unit_lens)} unit lengths")
        if len(text_lens) > 65535:
            raise ValueError(f"batch of {len(text_lens)} rows exceeds the kernels' limit of 65535 rows per launch")
        if max(text_lens) > MAX_TEXT:
            raise ValueError(f"a text of {max(text_lens)} characters exceeds the alignment search's limit of {MAX_TEXT}")
        rows = len(text_lens) * (max(max(text_lens), max(unit_lens)) + 2)
        if (rows + 127) // 128 > GEMM_MAX_ROW_TILES:
            raise ValueError(f"batch needs {(rows + 127) // 128} row tiles in one sb_gemm launch; the limit is "
                             f"{GEMM_MAX_ROW_TILES} (65535 x 128 rows): split the batch")

    @torch.inference_mode()
    def forward(self, text_ids: torch.Tensor, unit_ids: torch.Tensor, text_lens, unit_lens,
                marks: Optional[List[torch.cuda.Event]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """text_ids (B, T_text) character ids and unit_ids (B, T_feat) unit-vocabulary ids (already tokenised: u + 4),
        row b valid up to text_lens[b] / unit_lens[b] -> attn_lprob (B, max unit_lens, max text_lens) fp32 and durations
        (B, max text_lens) int64 on the device.  Row b equals that row run alone, bit for bit, in its [:F_b, :N_b] corner;
        padded tokens are -inf, padded frames 0, padded durations 0.  marks (timing tools): four CUDA events recorded once
        the ids and lengths are on the device (after the host-side checks and copies), then after the embeddings + convs,
        sb_align_lprob and sb_monotonic_align."""
        cfg, dev = self.cfg, self.device
        tl, ul = _as_list(text_lens), _as_list(unit_lens)
        self.check_batch(tl, ul)
        tids = self._ids(text_ids, tl, cfg.text_vocab_size, "text")
        uids = self._ids(unit_ids, ul, cfg.unit_vocab_size, "unit")
        tlens = torch.tensor(tl, dtype=I32, device=dev)
        ulens = torch.tensor(ul, dtype=I32, device=dev)
        if marks is not None:
            marks[0].record()
        t = self._convs(self._embed(tids, tlens, self.embed_text), self.t_conv)
        f = self._convs(self._embed(uids, ulens, self.embed_unit), self.f_conv)
        if marks is not None:
            marks[1].record()
        lprob = ops.align_lprob(f, t, cfg.temperature)
        if marks is not None:
            marks[2].record()
        dur = ops.monotonic_align(lprob, ulens, tlens)
        if marks is not None:
            marks[3].record()
        return lprob, dur.long()
