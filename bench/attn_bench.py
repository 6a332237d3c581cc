"""wgmma attention kernels vs torch SDPA (cuDNN flash) on the training shapes. CUDA events, L2 flushed between launches.

    python bench/attn_bench.py [OUT.json]

The first three rows are the head_dim <= 64 models; the others are the wider heads that `--attention native` runs on the
same kernels (llama_3b hd 80, llama_7b hd 128, Pythia-1.4B hd 128 and Pythia-1B hd 256 at the NeoX recipe's T = 2049).
FLOPs count the true head_dim, not the 64-column panels the kernels pad it to.  The card name, power limit and maximum SM
clock (read-only nvidia-smi query) are recorded with the rows."""
import math, os, subprocess, sys, json, torch
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

def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": clock, "torch": torch.__version__}

gpu = gpu_info()
print(json.dumps(gpu), flush=True)
rows = []
for name, B, T, nh, hd in (("250m", 24, 512, 16, 48), ("1b", 16, 512, 32, 64), ("1b_t2048", 4, 2048, 32, 64),
                           ("llama_3b", 16, 512, 32, 80), ("llama_7b", 4, 2048, 32, 128),
                           ("pythia_1.4b", 8, 2049, 16, 128), ("pythia_1b", 8, 2049, 8, 256)):
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
    json.dump({"gpu": gpu, "rows": rows}, open(sys.argv[1], "w"), indent=1)
