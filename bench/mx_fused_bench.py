"""`--quantize 8bit` on the fused Llama executor: tokens/s of fused-MX, module-MX and fused-bf16 in one process, alternating after
warm-up; gemm_mx against the bf16 wgmma GEMM at each projection and input-gradient shape (L2 flushed); resident frozen-weight
bytes of each executor.  Prints one JSON line per result; the card's name and power limit are read in the same run.

    python bench/mx_fused_bench.py [--models llama_250m llama_1b] [--train llama_250m] [--steps 6] [--rounds 3] [--parent-so PATH]

``--parent-so``: an extension built from an earlier commit (``relora_b200/csrc/build.py`` in its checkout); its gemm_mx is timed at
the same shapes, alternating with this one, and the outputs of the two on the same inputs are compared bit for bit.
(llama_1b's 5461-wide MLP is refused by the executor: the module path keeps such weights in a layout the tensor cores do not read.)
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

from gqa_bench import timeit  # noqa: E402
from pythia_bench import gpu_info  # noqa: E402

ROOT = os.path.dirname(HERE)
BF = torch.bfloat16
# micro-batch shapes of bench.py's workloads: llama_250m 48 x 256 tokens, llama_1b 32 x 256
SHAPES = {"llama_250m": (48, 256), "llama_1b": (32, 256)}


def build(name, quantize, seed=0):
    from relora_b200.models import LlamaForCausalLM, load_config
    from relora_b200.relora import ReLoRaModel

    torch.manual_seed(seed)
    cfg = load_config(os.path.join(ROOT, "configs", f"{name}.json"))
    m = ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "mlp"],
                    init_lora_a="kaiming", quantize=quantize)
    return m.cuda().to(BF)


def info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def stepper(kind, model):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    if kind == "module-mx":
        return ModuleStepper(model, info(), lr=1e-4, native=fused.NativeOptim())
    return FusedLlamaStepper(model, info(), lr=1e-4, quantize="mxfp8" if kind == "fused-mx" else None)


def frozen_bytes(kind, st):
    if kind == "fused-bf16":
        return sum(t.numel() * t.element_size() for t in (st.Wqkv, st.Wo, st.Wgu, st.Wd))
    if kind == "fused-mx":
        return sum(s.nbytes for stacks in st.Wmx for s in stacks)
    return sum(m.frozen_weight_nbytes() for m in st.model.relora_modules())


def train_rounds(name, steps, rounds):
    B, T = SHAPES[name]
    kinds = ("fused-mx", "module-mx", "fused-bf16")
    sts = {}
    for k in kinds:
        gc.collect()
        torch.cuda.empty_cache()
        m0 = torch.cuda.memory_allocated()
        sts[k] = stepper(k, build(name, None if k == "fused-bf16" else "mxfp8"))
        torch.cuda.synchronize()
        print(json.dumps({"model": name, "executor": k, "frozen_weight_bytes": frozen_bytes(k, sts[k]),
                          "allocated_after_construction": torch.cuda.memory_allocated() - m0}), flush=True)
    ids = torch.randint(0, 32000, (B, T), generator=torch.Generator().manual_seed(1)).cuda()
    for k in kinds:  # warm-up: graph capture, tensor maps, allocator
        for _ in range(2):
            sts[k].micro_step(ids)
            sts[k].update()
    torch.cuda.synchronize()
    rates = {k: [] for k in kinds}
    for _ in range(rounds):
        for k in kinds:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                loss = sts[k].micro_step(ids)
                sts[k].update()
            torch.cuda.synchronize()
            rates[k].append(B * T * steps / (time.perf_counter() - t0))
            assert torch.isfinite(loss), (k, float(loss))
    for k in kinds:
        print(json.dumps({"model": name, "executor": k, "tokens_per_s": sorted(rates[k]), "B": B, "T": T, "r": 128, "dropout": 0.1}),
              flush=True)
    del sts
    gc.collect()
    torch.cuda.empty_cache()


def gemm_rows(name, P=None):
    """gemm_mx (forward: K-major weight; input gradient: the same bytes MN-major) against fused.gemm in bf16, operands ready."""
    from relora_b200.models import load_config
    from relora_b200.ops import fused, mx

    C = fused._C()
    cfg = load_config(os.path.join(ROOT, "configs", f"{name}.json"))
    B, T = SHAPES[name]
    M, h, f = B * T, cfg.hidden_size, (cfg.intermediate_size + 127) // 128 * 128
    flush = torch.empty(64 * 2**20, dtype=torch.float32, device="cuda")  # 256 MB, past the 50 MB L2
    for site, N, K in (("qkv", 3 * h, h), ("o", h, h), ("gate|up", 2 * f, h), ("down", h, f)):
        g = torch.Generator(device="cuda").manual_seed(N + K)
        x = torch.randn(M, K, generator=g, device="cuda").to(BF)
        w = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(BF)
        dy = torch.randn(M, N, generator=g, device="cuda").to(BF)
        mw, (xq, sfx), (dq, sfd) = mx.quantize_weight(w), mx.quantize_rows(x), mx.quantize_rows(dy)
        y, dx = torch.empty(M, N, dtype=BF, device="cuda"), torch.empty(M, K, dtype=BF, device="cuda")
        fl = 2.0 * M * N * K
        row = {}
        if P is not None:  # the same calls on the earlier build's kernel, alternating, then the outputs compared bit for bit
            y0, dx0 = torch.empty_like(y), torch.empty_like(dx)
            tp = {}
            for k in ("fwd", "dx"):
                cur = (lambda: C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y, M, N, K, False)) if k == "fwd" else \
                      (lambda: C.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx, M, K, N, True))
                old = (lambda: P.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y0, M, N, K, False, None, None, None)) if k == "fwd" else \
                      (lambda: P.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx0, M, K, N, True, None, None, None))
                a, b = [], []
                for _ in range(3):
                    a.append(timeit(cur, flush))
                    b.append(timeit(old, flush))
                tp[f"mx_{k}_us_runs"], tp[f"parent_mx_{k}_us_runs"] = [round(v, 1) for v in a], [round(v, 1) for v in b]
            torch.cuda.synchronize()
            row = {**tp, "fwd_bit_identical": bool(torch.equal(y.view(torch.int16), y0.view(torch.int16))),
                   "dx_bit_identical": bool(torch.equal(dx.view(torch.int16), dx0.view(torch.int16)))}
        t = {
            "mx_fwd": timeit(lambda: C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y, M, N, K, False), flush),
            "bf16_fwd": timeit(lambda: fused.gemm(x, w, y, M=M, N=N, K1=K), flush),
            "mx_dx": timeit(lambda: C.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx, M, K, N, True), flush),
            "bf16_dx": timeit(lambda: fused.gemm(dy, w, dx, M=M, N=K, K1=N, b1_mn=True), flush),
        }
        print(json.dumps({"model": name, "site": site, "M": M, "N": N, "K": K,
                          **{f"{k}_us": round(v, 1) for k, v in t.items()},
                          **{f"{k}_tflops": round(fl / v / 1e6, 1) for k, v in t.items()}, **row}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["llama_250m", "llama_1b"])
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--train", nargs="*", default=["llama_250m"])
    ap.add_argument("--parent-so", default=None)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    P = None
    if a.parent_so:
        import importlib.util

        spec = importlib.util.spec_from_file_location("parent_build._C", a.parent_so)
        P = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(P)
    for name in a.models:
        gemm_rows(name, P)
    for name in a.train:
        train_rounds(name, a.steps, a.rounds)


if __name__ == "__main__":
    main()
