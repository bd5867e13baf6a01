"""The select half of a search step (sb_ban_step -> top-K -> sb_beam_step), which every search of the project runs:
the text search, the v1 unit search, MinTox re-decodes and the transcriber.

- All four top-K entry points (two-pass and per-tile statistics, each with and without bans) against a float64 top-K of
  the same fp32 rows, at vocabularies on both sides of K + 2 tiles of 128 for every K, with ragged last tiles and
  vocabularies that are not a multiple of 4, K from 1 to 16 and K > V - 1.  The rows put PAD / UNK / EOS at the top,
  tie tokens exactly across a tile boundary, hold one spike per tile (only n_tiles values reach the tile threshold), hold
  -inf entries, and sit in rows strided past the vocabulary.
- The tile path with the statistics of the real projection epilogue (sb_gemm tile_stats).
- Ban exhaustion on the tile path: the maxima of (nearly) every tile banned.
- The integer half of the text and unit searches replayed bit-exact on UnityOracle.beam_search's logits.
- The tiny_v1 unit search with and without tile statistics.
- Argument checks, on the CPU."""
import ctypes as Ct
import math

import numpy as np
import pytest
import torch

from oracle.unity_oracle import UnityOracle
from seamless_communication_b200 import config as C, synthetic as S
from seamless_communication_b200.models.unity.model import t2u_decoder_config
from test_gpu_parity import _replay_search_on_logits
from test_mintox import _tile_stats, _topk
from test_v1_s2st import _prefix, ar_state_dict, unit_oracle, with_reachable_eos

dev = "cuda"
gpu = pytest.mark.gpu
SB_EINVAL = -1  # include/seamless_b200.h
PAD, EOS, UNK, PEN = 0, 3, 1, 0.5
TILE = 128


# ------------------------------------------------------------------------------------------------ float64 reference
def _ref(x, K, pad, eos, unk, pen, bans=()):
    """Top-K of one fp32 row x [V]: ids in (value desc, id asc) order among the finite candidates (PAD and banned ids
    removed, the UNK penalty subtracted in fp32 as the kernel does), then (-inf, 0) fill; lprobs against the float64
    log-sum-exp of the whole row; the lprob of EOS (-inf when banned)."""
    V = x.shape[0]
    cand = x.clone()
    cand[unk] = cand[unk] - pen
    cand[pad] = -math.inf
    if len(bans):
        cand[list(bans)] = -math.inf
    v = cand.double().numpy()
    order = [int(i) for i in np.lexsort((np.arange(V), -v))[:K] if v[i] > -math.inf]
    lse = torch.logsumexp(x.double(), 0).item()
    ids = order + [0] * (K - len(order))
    vals = [v[i] - lse for i in order] + [-math.inf] * (K - len(order))
    el = -math.inf if eos in bans else float(x[eos]) - lse
    return ids, vals, el


def _assert_matches(cv, ci, el, x, K, bans, what, pen=PEN):
    for r in range(x.shape[0]):
        ids, vals, e = _ref(x[r], K, PAD, EOS, UNK, pen, bans[r] if bans else ())
        assert ci[r].tolist() == ids, f"{what}, row {r}"
        got = cv[r].double()
        want = torch.tensor(vals, dtype=torch.float64)
        fin = torch.isfinite(want)
        assert torch.equal(torch.isfinite(got), fin) and (got[~fin] == -math.inf).all(), f"{what}, row {r}"
        assert ((got - want)[fin].abs() < 2e-5).all(), f"{what}, row {r}"
        if e == -math.inf:
            assert el[r].item() == -math.inf, f"{what}, row {r}"
        else:
            assert abs(el[r].item() - e) < 2e-5, f"{what}, row {r}"


# ------------------------------------------------------------------------------------------------ rows
def _spikes(V, g, lo=-12.0, hi=-8.0):
    """One large value per 128-token tile, every other value below the weakest tile's maximum: only n_tiles values reach
    the (K+2)-th largest tile maximum."""
    nt = (V + TILE - 1) // TILE
    x = lo + (hi - lo) * torch.rand(V, generator=g)
    peaks = torch.linspace(0.0, 4.0, nt)[torch.randperm(nt, generator=g)]
    for t in range(nt):
        w = min(TILE, V - t * TILE)
        x[t * TILE + int(torch.randint(0, w, (1,), generator=g))] = peaks[t]
    return x


def _rows(V, seed):
    """Six fp32 rows of V logits and the ban list of each (row 0's list is empty)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(6, V, generator=g) * 3
    # 1: PAD, UNK and EOS head the row
    top = x[1].max()
    x[1, PAD], x[1, UNK], x[1, EOS] = top + 3, top + 2, top + 1
    # 2: exact ties at the top across a tile boundary (across the middle of a row shorter than two tiles); 1 800 of them
    # at the large vocabularies, below the 2 048 candidates the kernels hold
    n_tie = 1800 if V >= 10000 else min(V - 1, 24)
    lo = max(0, min(V - n_tie, TILE - n_tie // 2 if V > TILE + n_tie else (V - n_tie) // 2))
    ties = list(range(lo, lo + n_tie))
    x[2, ties] = x[2].max() + 1
    # 3: one spike per tile
    x[3] = _spikes(V, g)
    # 4: -inf entries: a whole aligned float4 group, every 7th token and the last one, never a whole tile (the
    # projection epilogue cannot write one)
    x[4, 4:8] = -math.inf
    x[4, ::7] = -math.inf
    if (V - 1) % TILE:
        x[4, V - 1] = -math.inf
    # 5: a second one-spike row
    x[5] = _spikes(V, g, -20.0, -1.0)
    best = lambda r, n: [int(i) for i in x[r].argsort(descending=True, stable=True)[:n]]
    peak_ids = [int(i) for i in (x[3] >= 0).nonzero().flatten()]
    bans = [[],
            [EOS, best(1, 4)[-1]],                                        # EOS banned
            ties[:3] + [ties[-1]],
            sorted(peak_ids, key=lambda i: -float(x[3, i]))[:3],            # the three largest tile maxima
            best(4, 5) + [PAD, best(4, 1)[0]],                              # duplicates and PAD
            [i for i in best(5, 40) if i % 3 == 0]]
    return x, [sorted({i for i in b if i < V}) for b in bans]


def _device_rows(x, ld, bait=1.0e4):
    """x [R, V] in a row stride ld > V whose padding holds values that would win if they were read."""
    lg = torch.full((x.shape[0], ld), bait)
    lg[:, :x.shape[1]] = x
    return lg.to(dev)


VOCABS = [5, 37, 127, 128, 129, 338, 640, 1126, 2175, 2176, 2305, 10082, 256102]


@gpu
@pytest.mark.parametrize("K", [1, 3, 11, 15, 16])
@pytest.mark.parametrize("V", VOCABS)
def test_topk_entry_points_match_float64(V, K):
    """sb_logits_topk, sb_logits_topk_ban, sb_logits_topk_tiles and sb_logits_topk_tiles_ban against the float64 top-K of
    the same rows: ids in (lprob desc, id asc) order, lprobs within 2e-5 of x - logsumexp64, eos_lprob, -inf / 0 fill
    past the candidates.  The tile and two-pass paths return the same ids, and an empty ban list equals the unbanned
    entry bit for bit.  A UNK penalty of -12 lifts UNK from the bottom of the one-spike rows to among their tile maxima."""
    x, bans = _rows(V, 1000 * V + K)
    ld = (V // 4 + 2) * 4
    lg = _device_rows(x, ld)
    for pen in (PEN, -12.0):
        out = {}
        for tiles in (False, True):
            for ban in (False, True):
                what = f"V={V} K={K} unk_penalty={pen} tiles={tiles} ban={ban}"
                cv, ci, el = out[tiles, ban] = _topk(lg, V, K, PAD, EOS, UNK, pen, bans=bans if ban else None, tiles=tiles)
                _assert_matches(cv, ci, el, x, K, bans if ban else None, what, pen)
            assert all(torch.equal(a[0], b[0]) for a, b in zip(out[tiles, True], out[tiles, False])), f"tiles={tiles}"
        for ban in (False, True):
            assert torch.equal(out[False, ban][1], out[True, ban][1]), f"V={V} K={K} ban={ban}: tile and two-pass ids differ"


@gpu
@pytest.mark.parametrize("V", [129, 1126, 2305, 10082])
def test_topk_tiles_on_projection_epilogue_statistics(V):
    """The tile path on logits and statistics written by sb_gemm(tile_stats=...): identity activations turn the fp16
    weight columns into exactly the wanted fp32 logits (random and one-spike rows), so the float64 reference knows
    them."""
    from seamless_communication_b200.ops import Seq, gemm
    R, D = 6, 64
    g = torch.Generator().manual_seed(V)
    want = torch.randn(R, V, generator=g) * 3
    want[1] = _spikes(V, g)
    want[2] = _spikes(V, g, -9.0, -2.0)
    want[3, 300 % V: 300 % V + 20] = want[3].max() + 1  # exact ties
    want = want.half().float()
    a = Seq(1, R, D, buf=torch.eye(R, D).half().to(dev))
    w = torch.zeros(V, D).half()
    w[:, :R] = want.t().half()
    ld = (V + 7) // 8 * 8
    logits = Seq(1, R, V, dtype=torch.float32, buf=torch.full((R, ld), float("nan"), device=dev))
    stats = torch.full(((V + TILE - 1) // TILE, R, 2), float("nan"), device=dev)
    gemm(a, w.to(dev), V, None, out=logits, out_f32=True, tile_stats=stats)
    assert torch.equal(logits.buf[:, :V].cpu(), want)
    bans = [[], [EOS], [int(want[2].argmax())], [], [1, 2, 3], []]
    for K in (1, 3, 11, 16):
        for b in (None, bans):
            cv, ci, el = _topk(logits.buf, V, K, PAD, EOS, UNK, PEN, bans=b, tiles=True, stats=stats)
            _assert_matches(cv, ci, el, want, K, b, f"V={V} K={K} bans={b is not None}")


@gpu
def test_ban_exhaustion_on_the_tile_path():
    """V = 20 102 (157 full tiles and a ragged one), K = 11: the maxima of all full tiles but K + 1, all but K, and all
    of them banned.  Fewer than K + 2 tiles then have a maximum that is not banned; the answer is still the float64
    top-K, on both paths, and the same on a second run."""
    V, K, R = 20102, 11, 3
    g = torch.Generator().manual_seed(20102)
    x = torch.randn(R, V, generator=g) * 3
    full = V // TILE
    tmax = (x[:, :full * TILE].reshape(R, full, TILE).argmax(-1) + torch.arange(full) * TILE).tolist()
    keep = torch.randperm(full, generator=g).tolist()
    bans = [sorted(tmax[0][t] for t in keep[K + 1:]), sorted(tmax[1][t] for t in keep[K:]), sorted(tmax[2])]
    lg = _device_rows(x, (V + 7) // 8 * 8)
    for tiles in (False, True):
        first = _topk(lg, V, K, PAD, EOS, UNK, PEN, bans=bans, tiles=tiles)
        _assert_matches(*first, x, K, bans, f"tiles={tiles}")
        again = _topk(lg, V, K, PAD, EOS, UNK, PEN, bans=bans, tiles=tiles)
        assert all(torch.equal(a, b) for a, b in zip(first, again)), f"tiles={tiles}: runs differ"


# ------------------------------------------------------------------------------------------------ search replay
# Each search runs twice: on the synthetic weights, which score EOS 0 so that every hypothesis ends on the forced EOS,
# and with an EOS row scaled to end hypotheses at different lengths (where the length penalty decides).  A negative UNK
# penalty lifts UNK, otherwise hundreds of places down these rows, into the candidate lists.
_SEARCH = {"text": dict(unk_penalty=-11.0, eos_scales=(0.0, 3.0)), "units": dict(unk_penalty=-12.0, eos_scales=(0.0, 1.5))}
_TRACES = {}


def _oracle_trace(kind, beam, len_penalty, eos_scale):
    key = (kind, beam, len_penalty, eos_scale)
    if key not in _TRACES:
        if kind == "text":
            cfg = C.tiny_v2()
            sd, toks = S.make_unity_state_dict(cfg, 0, dec_gain=4.0), S.make_tokenizers(cfg)
            if eos_scale:
                sd = with_reachable_eos(sd, cfg, eos_scale, text=True)
            oracle, dcfg = UnityOracle(cfg.to_dict(), sd, toks), cfg
            prefix, soft, hard = [cfg.text_eos, toks[0].lang_index("spa")], (1, 200), 30
        else:
            cfg = C.tiny_v1()
            sd = ar_state_dict()
            if eos_scale:
                sd = with_reachable_eos(sd, cfg, eos_scale)
            oracle, dcfg = unit_oracle(cfg, sd), t2u_decoder_config(cfg)
            prefix, soft, hard = _prefix(cfg), (25, 50), 40
        torch.manual_seed(17 + beam)
        enc = torch.randn(1, 11, cfg.model_dim)
        trace = {"sentence": 0}
        with torch.inference_mode():
            oracle.beam_search(enc, None, prefix, beam=beam, soft_max=soft, hard_max=hard, len_penalty=len_penalty,
                               unk_penalty=_SEARCH[kind]["unk_penalty"], trace=trace)
        _TRACES[key] = (dcfg, prefix, trace)
    return _TRACES[key]


@gpu
@pytest.mark.parametrize("len_penalty", [1.0, 0.5])
@pytest.mark.parametrize("tiles", [False, True])
@pytest.mark.parametrize("beam", [1, 2, 5, 7])
@pytest.mark.parametrize("kind", ["text", "units"])
def test_search_replay_is_bit_exact_on_oracle_logits(kind, beam, tiles, len_penalty):
    """Top-K (either path) -> sb_beam_step -> sb_step_advance on UnityOracle.beam_search's own fp32 logits: the tiny_v2
    text search (1 126 tokens) and the tiny_v1 unit search (338 units), with a nonzero UNK penalty, EOS forced at the
    budget and EOS reachable.  Parents, tokens and the finished hypotheses in finalisation order equal the oracle's at
    every step."""
    for eos_scale in _SEARCH[kind]["eos_scales"]:
        cfg, prefix, trace = _oracle_trace(kind, beam, len_penalty, eos_scale)
        decisions, finished = _replay_search_on_logits(cfg, trace, prefix, beam, cfg.text_vocab, len_penalty=len_penalty,
                                                       tiles=tiles, unk_penalty=_SEARCH[kind]["unk_penalty"])
        what = f"EOS scale {eos_scale}"
        assert len(decisions) == len(trace["beam_idx"]), what
        for s, (parents, toks) in enumerate(decisions):
            assert parents == trace["beam_idx"][s].tolist(), f"{what}, step {s}: parent beams differ"
            if s + 1 < len(trace["inputs"]):
                assert toks == trace["inputs"][s + 1].tolist(), f"{what}, step {s}: tokens differ"
        assert [f[1] for f in finished] == [f[1] for f in trace["finished"]], what
        assert np.allclose([f[0] for f in finished], [f[0] for f in trace["finished"]], rtol=0, atol=1e-5), what


@gpu
def test_unit_search_same_with_and_without_tile_statistics(monkeypatch):
    """The tiny_v1 unit search (338 units: fewer than K + 2 tiles at every beam) gives the same hypotheses and scores,
    bit for bit, with SB_TOPK_TILES=0 and =1."""
    from seamless_communication_b200.models.unity import load_unity_model
    from seamless_communication_b200.ops import Seq
    cfg = C.tiny_v1()
    sd, toks = with_reachable_eos(ar_state_dict(), cfg, 1.5), S.make_tokenizers(cfg)
    t2u = {}
    for flag in ("0", "1"):
        monkeypatch.setenv("SB_TOPK_TILES", flag)
        t2u[flag] = load_unity_model("tiny_v1", state_dict=sd, tokenizers=toks).t2u_model
        assert t2u[flag].unit_engine.topk_tiles == (flag == "1")
    lens = [11, 6]
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 11, cfg.model_dim, generator=g)
    x[1, 6:] = 0
    enc = Seq(2, 11, cfg.model_dim, buf=x.view(22, -1).half().to(dev))
    el = torch.tensor(lens, dtype=torch.int32, device=dev)
    for beam in (1, 2, 5, 7):
        got = {f: m.beam_search(enc, el, _prefix(cfg), beam=beam, soft_max=(25, 50), hard_max=48, unk_penalty=-12.0)
               for f, m in t2u.items()}
        assert got["0"] == got["1"], f"beam {beam}"


# ------------------------------------------------------------------------------------------------ CPU: argument checks
_BASE = 1 << 24  # never dereferenced: every call below is refused before anything is launched


def _call(entry, ld=1128, ptr=_BASE, eos=EOS, V=1126):
    from seamless_communication_b200 import _lib
    lib = _lib.load()
    K, R = 11, 2
    out = dict(cv=_BASE + (1 << 20), ci=_BASE + (2 << 20), el=_BASE + (3 << 20))
    stats, ban_ids, ban_n = _BASE + (4 << 20), _BASE + (5 << 20), _BASE + (6 << 20)
    head = (ptr, ld) + ((stats,) if "tiles" in entry else ()) + (R, V, PAD, eos, UNK, PEN, K, out["cv"], out["ci"], out["el"])
    tail = (ban_ids, ban_n, 4) if entry.endswith("ban") else ()
    n0 = lib.sb_launch_count()
    rc = getattr(lib, entry)(*head, *tail, None)
    assert lib.sb_launch_count() == n0
    return rc, (lib.sb_last_error() or b"").decode()


ENTRIES = ["sb_logits_topk", "sb_logits_topk_ban", "sb_logits_topk_tiles", "sb_logits_topk_tiles_ban"]


@pytest.mark.parametrize("bad", ["ld", "align", "eos_high", "eos_neg"])
@pytest.mark.parametrize("entry", ENTRIES)
def test_topk_refuses_bad_arguments_before_any_cuda_call(entry, bad):
    """Rows the float4 loads cannot read (a row stride that is not a multiple of 4, logits not 16-byte aligned) and an
    EOS id outside the vocabulary return SB_EINVAL, with nothing launched."""
    kw = dict(ld=dict(ld=1127), align=dict(ptr=_BASE + 4), eos_high=dict(eos=1126), eos_neg=dict(eos=-1))[bad]
    rc, msg = _call(entry, **kw)
    assert rc == SB_EINVAL, (entry, bad, rc, msg)
    assert entry in msg
