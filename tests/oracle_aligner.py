"""CPU restatement of the UnitY2 aligner (reference models/aligner/model.py:146-277) in float64 torch / numpy, held to
tests/golden/aligner.npz (made by the reference's own code) in tests/test_aligner.py."""
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

TEXT_CONVS = ("t_conv.1", "t_conv.4")
FEAT_CONVS = ("f_conv.1", "f_conv.4", "f_conv.7")


def _convs(x: torch.Tensor, sd: Dict[str, torch.Tensor], names, prefix: str) -> torch.Tensor:
    """(T, C) -> (T, M): Conv1d(k3, pad 1) -> ReLU for all but the last, Conv1d(k1) last."""
    h = x.t()[None]
    for n, name in enumerate(names):
        w, b = sd[f"{prefix}{name}.weight"].to(h.dtype), sd[f"{prefix}{name}.bias"].to(h.dtype)
        h = F.conv1d(h, w, b, padding=w.shape[2] // 2)
        if n < len(names) - 1:
            h = F.relu(h)
    return h[0].t()


def encoder_lprob(sd, text_emb: torch.Tensor, feat_emb: torch.Tensor, temperature: float = 1.0, prefix: str = "",
                  ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """One row: text_emb (T_text, C), feat_emb (T_feat, C) -> lprob (T_feat, T_text), text states, feature states, in
    the inputs' dtype.  Distances are direct differences."""
    t = _convs(text_emb, sd, TEXT_CONVS, prefix)
    f = _convs(feat_emb, sd, FEAT_CONVS, prefix)
    return lprob_from_states(f, t, temperature), t, f


U16, U32 = 2.0 ** -11, 2.0 ** -24


def state_error_std(sd, emb: torch.Tensor, names, prefix: str = "") -> torch.Tensor:
    """Elementwise standard deviation of state - state64 for one branch run as the CUDA path runs it, modelling every
    rounding as an independent error uniform within half an ulp (variance (u |v|)^2 / 3 for a relative roundoff u):
    the fp16 embeddings and weights, the fp16 store of every intermediate conv output and the fp32 store of the last.
    A conv maps input error variances through w^2 (it is linear in its input); ReLU keeps at most the variance it is given.
    fp32 accumulation of the K = taps * c_in fp16 products rounds K partial sums, each at most sum |w||x| in size: a
    deviation of sqrt(K / 3) 2^-24 sum |w||x| under the same model."""
    x = emb.double()
    var = (emb.half().double() - x).pow(2)
    for n, name in enumerate(names):
        w = sd[f"{prefix}{name}.weight"].double()
        b = sd[f"{prefix}{name}.bias"].double()
        pad = w.shape[2] // 2
        dw = w.half().double() - w
        y = F.conv1d(x.t()[None], w, b, padding=pad)[0].t()
        K = w.shape[1] * w.shape[2]
        acc = (K / 3) ** 0.5 * U32 * F.conv1d(x.abs().t()[None], w.abs(), None, padding=pad)[0].t()
        var = (F.conv1d(var.t()[None], w.pow(2), None, padding=pad)[0].t()
               + F.conv1d(x.pow(2).t()[None], dw.pow(2), None, padding=pad)[0].t() + acc.pow(2))
        if n < len(names) - 1:
            y = F.relu(y)
            var = var * (y > 0) + (U16 * y).pow(2) / 3
        else:
            var = var + (U32 * y).pow(2) / 3
        x = y
    return var.sqrt()


def lprob_error_bound(f: torch.Tensor, t: torch.Tensor, sf: torch.Tensor, st: torch.Tensor, temperature: float,
                      ref: torch.Tensor, k: float = 6.0) -> torch.Tensor:
    """Bound on |lprob - lprob64| (T_feat, T_text) at k standard deviations of the state errors (sf / st from
    state_error_std): to first order a distance moves by the state errors projected on the unit difference
    (f_j - t_i) / d_ji, so the score's deviation is sigma_ji = temperature * sqrt(sum_c r_c^2 (sf_jc^2 + st_ic^2)); the
    log-sum-exp moves by a p-weighted mean of the score errors, at most max_i of them.  Added deterministically: the fp32
    distance ((dim + 5)/2 2^-24 d), the fp32 exp / sum / log roundings (4 u (|lse| + max|s|) + 4 N u) and the fp32 store
    of the result (u |lp|)."""
    dim, N = f.shape[1], t.shape[0]
    rows = []
    for j in range(0, f.shape[0], 64):
        diff = f[j:j + 64, None, :] - t[None, :, :]
        d = diff.pow(2).sum(-1).sqrt()
        r2 = diff.pow(2) / d.clamp_min(1e-300)[..., None].pow(2)
        sig = (r2 * (sf[j:j + 64, None, :].pow(2) + st[None, :, :].pow(2))).sum(-1).sqrt()
        rows.append((d, sig))
    d = torch.cat([r[0] for r in rows])
    sig = temperature * torch.cat([r[1] for r in rows])
    E = k * sig + temperature * (dim + 5) / 2 * U32 * d
    s = -temperature * d
    lse = torch.logsumexp(s, -1, keepdim=True)
    return E + E.max(-1, keepdim=True).values + 4 * U32 * (lse.abs() + s.abs().max(-1, keepdim=True).values) + 4 * N * U32 \
        + U32 * ref.abs()


def lprob_from_states(f: torch.Tensor, t: torch.Tensor, temperature: float = 1.0) -> torch.Tensor:
    """log_softmax over tokens of -temperature * ||f_j - t_i||, 64 frames at a time (the difference tensor is large)."""
    dist = torch.cat([(f[j:j + 64, None, :] - t[None, :, :]).pow(2).sum(-1).sqrt() for j in range(0, f.shape[0], 64)])
    return torch.log_softmax(-temperature * dist, -1)


def mas_q(lp: np.ndarray, numpy_row0: bool = False) -> np.ndarray:
    """Q (T_text, T_feat) float64 of the alignment search on lp (T_feat, T_text) float32.  Row 0 is a float64 running
    sum (the CUDA kernel's order); numpy_row0 takes numpy's float32 sum of the prefix instead, as the reference does."""
    lp = np.asarray(lp, dtype=np.float32)
    T_feat, T_text = lp.shape
    Q = np.full((T_text, T_feat), -np.inf)
    if numpy_row0:
        Q[0] = [lp[:j + 1, 0].sum() for j in range(T_feat)]
    else:
        Q[0] = np.cumsum(lp[:, 0].astype(np.float64))
    for j in range(1, T_feat):
        m = min(j, T_text - 1)
        if m >= 1:
            Q[1:m + 1, j] = np.maximum(Q[0:m, j - 1], Q[1:m + 1, j - 1]) + lp[j, 1:m + 1].astype(np.float64)
    return Q


def mas_path(lp: np.ndarray, numpy_row0: bool = False, Q: Optional[np.ndarray] = None) -> np.ndarray:
    Q = mas_q(lp, numpy_row0) if Q is None else Q
    T_text, T_feat = Q.shape
    A = np.full((T_feat,), T_text - 1)
    for j in range(T_feat - 2, -1, -1):
        ib = A[j + 1]
        A[j] = 0 if ib == 0 else (ib - 1 if Q[ib - 1, j] >= Q[ib, j] else ib)
    return A


def durations(lp: np.ndarray, numpy_row0: bool = False) -> np.ndarray:
    lp = np.asarray(lp)
    return np.bincount(mas_path(lp, numpy_row0), minlength=lp.shape[1])


def decision_margins(lp: np.ndarray) -> np.ndarray:
    """|Q[i-1][j] - Q[i][j]| of every decision the backtrack takes (inf where it is forced), per column j < T_feat - 1."""
    Q = mas_q(lp)
    A = mas_path(lp, Q=Q)
    out = np.full(len(A) - 1, np.inf)
    for j in range(len(A) - 1):
        ib = A[j + 1]
        if 0 < ib <= j:
            out[j] = abs(Q[ib - 1, j] - Q[ib, j])
    return out


def forward(sd: Dict[str, torch.Tensor], text_ids: torch.Tensor, unit_ids: torch.Tensor, temperature: float = 1.0,
            dtype=torch.float64):
    """UnitY2AlignmentModel.forward for one row of ids under the model's names -> lprob (T_feat, T_text), durations."""
    te = sd["alignment_frontend.embed_text.weight"].to(dtype)[text_ids]
    ue = sd["alignment_frontend.embed_unit.weight"].to(dtype)[unit_ids]
    lp, _, _ = encoder_lprob(sd, te, ue, temperature, prefix="alignment_encoder.")
    return lp, durations(lp.float().numpy())
