"""Run the wgmma attention kernels a few times (a short, profiler-friendly workload)."""
import math, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relora_b200.ops import fused as F
C = F._C(); B, T, nh, hd = 24, 512, 16, 48; h = nh * hd
qkv = (torch.randn(B * T, 3 * h, device="cuda") * 0.5).bfloat16(); out = torch.empty(B * T, h, device="cuda", dtype=torch.bfloat16)
lse = torch.empty(B, nh, T, device="cuda", dtype=torch.float32); delta = torch.empty_like(lse); dout = torch.randn_like(out); dqkv = torch.empty_like(qkv)
ws = torch.empty(C.attention_ds_workspace_elems(B, T, nh), device="cuda", dtype=torch.bfloat16)  # dS-store backward (the executor's default)
for _ in range(4):
    C.attention_fwd(qkv, out, lse, B, T, nh, hd, 1 / math.sqrt(hd)); C.attention_bwd(qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, 1 / math.sqrt(hd), ws)
torch.cuda.synchronize(); print("ok")
