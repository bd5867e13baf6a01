"""The weight-stationary vocabulary projection (vocab_proj_kernel in decode_gemm.cu): sb_gemm with tile_stats at <= 256
rows.  Its logits and per-tile log-softmax statistics must equal those of the general kernel (SB_PROJ_T=0) bit for
bit, since a last-bit change in a row's log-sum-exp shifts every candidate of the row and can flip a cross-beam near
tie, and agree with the CUDA-core reference kernel within fp32 summation-order noise."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"


def _project(ops, a, w, V, proj_t):
    from seamless_communication_b200.ops import Seq
    R = a.buf.shape[0]
    ld = (V + 7) // 8 * 8
    logits = Seq(1, R, V, dtype=torch.float32, buf=torch.full((R, ld), float("nan"), device=dev))
    stats = torch.full(((V + 127) // 128, R, 2), float("nan"), device=dev)
    old = os.environ.get("SB_PROJ_T")
    os.environ["SB_PROJ_T"] = "1" if proj_t else "0"
    try:
        ops.gemm(a, w, V, None, out=logits, out_f32=True, tile_stats=stats)
    finally:
        if old is None:
            del os.environ["SB_PROJ_T"]
        else:
            os.environ["SB_PROJ_T"] = old
    torch.cuda.synchronize()
    return logits.buf[:, :V], stats


@pytest.fixture(scope="module")
def ops():
    from seamless_communication_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def embedding():
    torch.manual_seed(11)
    return (torch.randn(256102, 1024, device=dev) * 0.05).half()


@pytest.mark.parametrize("R,V", [(160, 256102), (37, 256102), (5, 256102), (256, 256102), (160, 3001)])
def test_vocab_projection_matches_general_kernel_and_reference(ops, embedding, R, V):
    from seamless_communication_b200.ops import Seq
    torch.manual_seed(R + V)
    a = Seq(1, R, 1024, buf=torch.randn(R, 1024, device=dev).half())
    w = embedding[:V]
    new_l, new_s = _project(ops, a, w, V, True)
    old_l, old_s = _project(ops, a, w, V, False)
    assert torch.isfinite(new_l).all() and torch.isfinite(new_s).all()
    d = (new_l - old_l).abs().max().item()
    assert torch.equal(new_l, old_l), f"logits differ from the general kernel's by up to {d:.3g}"
    assert torch.equal(new_s, old_s), "tile statistics differ from the general kernel's"
    ref = ops.gemm_raw(a.buf, w, V, out_f32=True, ref=True)
    assert (new_l - ref).abs().max().item() < 1e-4 * ref.abs().max().item()  # summation order and tensor-core rounding only
    # the statistics describe the logits that were stored
    tiles = new_l.new_full((R, new_s.shape[0] * 128), -math.inf)
    tiles[:, :V] = new_l
    tiles = tiles.view(R, -1, 128)
    assert torch.equal(new_s[:, :, 0].t(), tiles.max(-1).values)
    assert torch.allclose(new_s[:, :, 1].t(), torch.exp(tiles - tiles.max(-1, keepdim=True).values).sum(-1), rtol=1e-5)

