"""T(K) sweep at fixed M, N: separates the per-tile fixed cost (epilogue, tile hand-off) from the per-k-block cost
(tensor pipe / L2 feed) for the 128-, 192- and 256-wide tiles of the wgmma GEMM, the 128-wide one also as CTA pairs.

    python bench/gemm_ksweep.py [--M 12288] [--N 2304] [--out gemm_ksweep.json]
"""
import argparse, json, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from relora_b200.ops import fused as F


def timeit(fn, flush, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    ts.sort()
    return ts[len(ts) // 2]


ap = argparse.ArgumentParser()
ap.add_argument("--M", type=int, default=12288); ap.add_argument("--N", type=int, default=2304); ap.add_argument("--out", default=None)
a = ap.parse_args()
flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
rows = []
for K in (128, 256, 512, 768, 1536, 3072, 6144):
    x = torch.randn(a.M, K, device="cuda").bfloat16(); W = (torch.randn(a.N, K, device="cuda") * 0.02).bfloat16()
    out = torch.empty(a.M, a.N, device="cuda", dtype=torch.bfloat16)
    outf = torch.zeros(a.M, a.N, device="cuda", dtype=torch.float32)
    rec = {"M": a.M, "N": a.N, "K": K}
    rec["cublas_us"] = timeit(lambda: torch.matmul(x, W.t(), out=out), flush) * 1e6
    rec["bn128_us"] = timeit(lambda: F.gemm(x, W, out, block_n=128, pair=0), flush) * 1e6
    rec["bn192_us"] = timeit(lambda: F.gemm(x, W, out, block_n=192, pair=0), flush) * 1e6
    rec["bn128_pair_us"] = timeit(lambda: F.gemm(x, W, out, block_n=128, pair=1), flush) * 1e6
    rec["bn256_us"] = timeit(lambda: F.gemm(x, W, out, block_n=256, pair=0), flush) * 1e6
    rec["pair_us"] = timeit(lambda: F.gemm(x, W, out, block_n=256, pair=1), flush) * 1e6
    # fp32 accumulate output: stored from registers (global read-modify-write), the epilogue of the weight gradients
    rec["bn256_f32acc_us"] = timeit(lambda: F.gemm(x, W, outf, block_n=256, pair=0, accumulate=True), flush) * 1e6
    rows.append(rec)
    print(json.dumps({k: (round(v, 1) if isinstance(v, float) else v) for k, v in rec.items()}), flush=True)
if a.out:
    json.dump(rows, open(a.out, "w"), indent=1)
