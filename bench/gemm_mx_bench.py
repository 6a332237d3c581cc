"""Block-scaled MXFP8 GEMM (csrc/gemm_mx.cu) vs the bf16 wgmma GEMM on the model's projection shapes; operands pre-quantised.

    python bench/gemm_mx_bench.py [--out gemm_mx_bench.json]
"""
import argparse, json, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relora_b200.ops import fused as F, mx
ap = argparse.ArgumentParser(); ap.add_argument("--out", default=None); ap.add_argument("--iters", type=int, default=20); a = ap.parse_args()
C = F._C(); rows = []
def timed(fn):
    for _ in range(3): fn()
    torch.cuda.synchronize(); e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters): fn()
    e1.record(); torch.cuda.synchronize(); return e0.elapsed_time(e1) / a.iters * 1e3
for tag, M, N, K in (("250m qkv", 12288, 2304, 768), ("250m gate/up", 12288, 5120, 768), ("250m down", 12288, 768, 2560),
                     ("1b qkv", 8192, 6144, 2048), ("1b gate/up", 8192, 11008, 2048), ("1b down", 8192, 2048, 5504)):
    x = (torch.randn(M, K, device="cuda")).bfloat16(); w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    mw = mx.quantize_weight(w); xq, sfx = mx.quantize_rows(x); y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    t_mx = timed(lambda: C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y, M, N, K, False, None, None, None))
    t_q = timed(lambda: mx.quantize_rows(x))
    yb = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    t_bf = timed(lambda: F.gemm(x, w, yb, M=M, N=N, K1=K))
    dy = torch.randn(M, N, device="cuda").bfloat16(); dq, sfd = mx.quantize_rows(dy); dx = torch.empty(M, K, device="cuda", dtype=torch.bfloat16)
    t_dx = timed(lambda: C.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx, M, K, N, True, None, None, None))
    fl = 2.0 * M * N * K
    rec = {"site": tag, "M": M, "N": N, "K": K, "mx_fwd_us": t_mx, "mx_fwd_tflops": fl / t_mx / 1e6, "mx_dx_us": t_dx, "mx_dx_tflops": fl / t_dx / 1e6,
           "bf16_us": t_bf, "bf16_tflops": fl / t_bf / 1e6, "quantize_rows_us": t_q, "weight_bytes_ratio": mw.nbytes / (2.0 * N * K)}
    rows.append(rec); print(json.dumps(rec), flush=True)
if a.out:
    os.makedirs(os.path.dirname(a.out), exist_ok=True); json.dump(rows, open(a.out, "w"), indent=1)
