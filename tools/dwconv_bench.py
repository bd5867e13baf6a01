import sys, torch, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from seamless_communication_b200 import ops
from seamless_communication_b200.ops import Seq
torch.manual_seed(0)
B, T, C, k = 32, 499, 1024, 31
x = Seq(B, T, C, buf=(torch.randn(B * T, C, device="cuda") * 0.5).half())
w = (torch.randn(C, k, device="cuda") * 0.2).half()
lw, lb = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.1
import torch.nn.functional as F
def run(): return ops.dwconv_ln_silu(x, w, lw, lb, k)
y = run()
c = F.conv1d(F.pad(x.buf.float().view(B, T, C).transpose(1, 2), (k - 1, 0)), w.float().view(C, 1, k), groups=C)
ref = F.silu(F.layer_norm(c.transpose(1, 2), (C,), lw, lb, 1e-5)).reshape(B * T, C)
print("max abs err", (y.buf.float() - ref).abs().max().item(), "rel", ((y.buf.float() - ref).abs().max() / ref.abs().max()).item())
for tag in ("tile", "old"):
    if tag == "old": os.environ["SB_DWCONV_TILE"] = "0"
    for _ in range(3): run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20): run()
    e1.record(); torch.cuda.synchronize()
    print(tag, e0.elapsed_time(e1) / 20 * 1e3, "us")
    break
