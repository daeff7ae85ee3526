"""Developer tool: error of the fp32-grade split GEMM vs fp64 for several accumulator run lengths."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from otter_b200 import functional as F
torch.manual_seed(0)
x = torch.randn(256, 1024, device="cuda"); w = torch.randn(512, 1024, device="cuda") / 32
ref = (x.double() @ w.double().t())
w6 = F.split3_concat(w, 1)
for kc in (1 << 20, 2048, 512, 128, 64):
    F.F32_KCHUNK = kc
    y = F.linear_f32(x, w6, 512)
    err = (y.double() - ref).abs()
    print(f"kchunk {kc:8d}: max abs err {err.max().item():.3e}  mean {err.mean().item():.3e}  (|ref| rms {ref.pow(2).mean().sqrt().item():.2f})")
y32 = x @ w.t()
print("torch fp32 matmul (TF32 off):", (y32.double() - ref).abs().max().item())
