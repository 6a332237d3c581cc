"""Per-kernel roofline bench: wgmma GEMM (plain / fused-LoRA / MN-major / split-K) vs cuBLAS via torch.matmul.

    python bench/gemm_bench.py [--out gemm_bench.json]

CUDA-event timing, 3 warm-up + 10 timed launches, a 256 MB write between launches flushes the 50 MB L2.
Fractions are reported against MEASURED_PEAKS.json (bf16_tflops burst) when present, else against the H100 SXM
data sheet's 989 TFLOP/s dense BF16.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from relora_b200.ops import fused as F  # noqa: E402

BF = torch.bfloat16


def peak_tflops():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops"]
    except Exception:
        return 989.0


def timeit(fn, flush, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--M", type=int, default=12288)
    a = ap.parse_args()
    dev = "cuda"
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    peak = peak_tflops()
    rows = []
    M = a.M
    shapes = [("qkv_250m", 2304, 768, 3), ("o_250m", 768, 768, 1), ("gateup_250m", 5120, 768, 2), ("down_250m", 768, 2560, 1),
              ("qkv_1b", 6144, 2048, 3), ("gateup_1b", 11008, 2048, 2), ("down_1b", 2048, 5504, 1), ("square_8k", 8192, 8192, 1)]
    for name, N, K, G in shapes:
        Mx = 8192 if name == "square_8k" else M
        x = torch.randn(Mx, K, device=dev).to(BF)
        W = (torch.randn(N, K, device=dev) * 0.02).to(BF)
        r = 128
        u = torch.randn(Mx, G * r, device=dev).to(BF)
        B = (torch.randn(N, r, device=dev) * 0.02).to(BF)
        out = torch.empty(Mx, N, device=dev, dtype=BF)
        flops = 2.0 * Mx * N * K
        t_cublas = timeit(lambda: torch.matmul(x, W.t(), out=out), flush)
        rec = {"shape": name, "M": Mx, "N": N, "K": K, "cublas_us": t_cublas * 1e6, "cublas_tflops": flops / t_cublas / 1e12}
        for bn in (128, 192, 256):
            try:
                t = timeit(lambda: F.gemm(x, W, out, block_n=bn, pair=0), flush)
                rec[f"ours_bn{bn}_us"] = t * 1e6
                rec[f"ours_bn{bn}_tflops"] = flops / t / 1e12
                rec[f"ours_bn{bn}_frac_of_measured_peak"] = flops / t / 1e12 / peak
            except Exception as e:  # keep benchmarking the other variants
                rec[f"ours_bn{bn}_error"] = str(e)[:200]
        try:
            t = timeit(lambda: F.gemm(x, W, out, block_n=128, pair=1), flush)
            rec["ours_pair_us"] = t * 1e6
            rec["ours_pair_tflops"] = flops / t / 1e12
            rec["ours_pair_frac_of_measured_peak"] = flops / t / 1e12 / peak
        except Exception as e:
            rec["ours_pair_error"] = str(e)[:200]
        if name != "square_8k":
            Ng = N // G
            bn = 256 if Ng % 256 == 0 else 128
            fl2 = flops + 2.0 * Mx * N * r
            t = timeit(lambda: F.gemm(x, W, out, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, block_n=bn, pair=0), flush)
            rec["ours_fused_lora_us"] = t * 1e6
            rec["ours_fused_lora_tflops"] = fl2 / t / 1e12
            t = timeit(lambda: F.gemm(x, W, out, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, block_n=128, pair=1), flush)
            rec["ours_fused_lora_pair_us"] = t * 1e6
            rec["ours_fused_lora_pair_tflops"] = fl2 / t / 1e12
            # what the reference does for the same math: F.linear + 2 small GEMMs + mul + add (no dropout here)
            def ref_path():
                y = torch.matmul(x, W.t())
                for g in range(G):
                    y[:, g * Ng:(g + 1) * Ng] += torch.matmul(u[:, g * r:(g + 1) * r], B[g * Ng:(g + 1) * Ng].t())
                return y
            t = timeit(ref_path, flush)
            rec["cublas_unfused_lora_us"] = t * 1e6
            # backward dx (B operand read MN-major from W[N,K])
            dy = torch.randn(Mx, N, device=dev).to(BF)
            dx = torch.empty(Mx, K, device=dev, dtype=BF)
            t = timeit(lambda: F.gemm(dy, W, dx, M=Mx, N=K, K1=N, b1_mn=True, pair=0), flush)
            rec["ours_dx_mnB_us"] = t * 1e6
            rec["ours_dx_mnB_tflops"] = flops / t / 1e12
            for bn in (128, 192):
                t = timeit(lambda: F.gemm(dy, W, dx, M=Mx, N=K, K1=N, b1_mn=True, block_n=bn, pair=0), flush)
                rec[f"ours_dx_mnB_bn{bn}_us"] = t * 1e6
            t = timeit(lambda: F.gemm(dy, W, dx, M=Mx, N=K, K1=N, b1_mn=True, block_n=128, pair=1), flush)
            rec["ours_dx_mnB_pair_us"] = t * 1e6
            rec["ours_dx_mnB_pair_tflops"] = flops / t / 1e12
            t = timeit(lambda: torch.matmul(dy, W, out=dx), flush)
            rec["cublas_dx_us"] = t * 1e6
            # LoRA weight grad: dB[N, r] = dyᵀ u (split-K over tokens)
            db = torch.zeros(N, G * r, device=dev, dtype=torch.float32)
            t = timeit(lambda: F.gemm(dy, u, db, M=N, N=G * r, K1=Mx, a1_mn=True, b1_mn=True, accumulate=True, split_k=0), flush)
            rec["ours_wgrad_splitk_us"] = t * 1e6
            t = timeit(lambda: torch.matmul(dy.t(), u), flush)
            rec["cublas_wgrad_us"] = t * 1e6
        rows.append(rec)
        print(json.dumps(rec), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        json.dump({"peak_tflops_measured": peak, "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
