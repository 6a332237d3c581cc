"""wgmma attention kernels vs torch SDPA (cuDNN flash) on the training shapes. CUDA events, L2 flushed between launches."""
import math, os, sys, json, torch
import torch.nn.functional as Fn
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relora_b200.ops import fused as F
C = F._C()
flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")

def timeit(fn, iters=10, warm=3):
    for _ in range(warm): fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort(); return ts[len(ts) // 2]

rows = []
for name, B, T, nh, hd in (("250m", 24, 512, 16, 48), ("1b", 16, 512, 32, 64), ("1b_t2048", 4, 2048, 32, 64)):
    h = nh * hd
    qkv = (torch.randn(B * T, 3 * h, device="cuda") * 0.5).bfloat16()
    out = torch.empty(B * T, h, device="cuda", dtype=torch.bfloat16)
    lse = torch.empty(B, nh, T, device="cuda", dtype=torch.float32)
    delta = torch.empty_like(lse)
    dout = (torch.randn(B * T, h, device="cuda") * 0.1).bfloat16()
    dqkv = torch.empty_like(qkv)
    sc = 1.0 / math.sqrt(hd)
    t_f = timeit(lambda: C.attention_fwd(qkv, out, lse, B, T, nh, hd, sc))
    t_b_recompute = timeit(lambda: C.attention_bwd(qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, sc))
    ws = torch.empty(C.attention_ds_workspace_elems(B, T, nh), device="cuda", dtype=torch.bfloat16)
    t_b = timeit(lambda: C.attention_bwd(qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, sc, ws))  # default: dS stored, dQ = dS·K
    v5 = qkv.view(B, T, 3, nh, hd)
    q, k, v = (v5[:, :, i].transpose(1, 2).detach().requires_grad_() for i in range(3))
    t_sf = timeit(lambda: Fn.scaled_dot_product_attention(q, k, v, is_causal=True))
    o = Fn.scaled_dot_product_attention(q, k, v, is_causal=True)
    g = dout.view(B, T, nh, hd).transpose(1, 2)
    t_sb = timeit(lambda: torch.autograd.grad(o, (q, k, v), g, retain_graph=True))
    fl = 4.0 * B * nh * T * T * hd / 2
    rec = {"shape": name, "B": B, "T": T, "nh": nh, "hd": hd, "ours_fwd_us": t_f, "sdpa_fwd_us": t_sf, "ours_bwd_us": t_b, "ours_bwd_recompute_us": t_b_recompute, "sdpa_bwd_us": t_sb,
           "ours_fwd_tflops": fl / t_f / 1e6, "ours_bwd_tflops": 2.5 * fl / t_b / 1e6}
    rows.append(rec); print(json.dumps({k: (round(x, 1) if isinstance(x, float) else x) for k, x in rec.items()}), flush=True)
if len(sys.argv) > 1:
    json.dump(rows, open(sys.argv[1], "w"), indent=1)
