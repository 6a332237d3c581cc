"""`--quantize 8bit` on the fused Pythia executor: tokens/s of fused-MX, module-MX and fused-bf16 in one process, alternating after
warm-up; gemm_mx with its bias epilogue against the bf16 wgmma GEMM with its bias at each projection shape (L2 flushed); resident
frozen-weight bytes of each executor.  Prints one JSON line per result; the card's name and power limit are read in the same run.

    python bench/pythia_mx_bench.py [--shapes 160m 410m 1b] [--steps 3] [--rounds 3] [--T 2049] [--parent-so PATH]

Random weights; ReLoRA r = 128, lora_dropout 0.1, T = 2049, the shapes and micro-batches of bench/pythia_bench.py.
``--parent-so``: an extension built from an earlier commit; its gemm_mx (no bias) runs on the same operands and the outputs are
compared bit for bit with this build's call without a bias.
"""
from __future__ import annotations

import argparse
import copy
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
from pythia_bench import SHAPES, gpu_info  # noqa: E402

BF = torch.bfloat16
KINDS = ("fused-mx", "module-mx", "fused-bf16")


def info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def build(name, quantize):
    """bench/pythia_bench.py's model at ``name``, its frozen weights packed when ``quantize`` is given."""
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    h, L, nh, f, _ = SHAPES[name]
    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=50304, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                       intermediate_size=f, rotary_pct=0.25, max_position_embeddings=2048, layer_norm_eps=1e-5,
                       use_parallel_residual=True, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    torch.manual_seed(0)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming", quantize=quantize)
    with torch.no_grad():
        for m in w.relora_modules():
            torch.nn.init.normal_(m.lora_B.weight, std=0.02)
    return w.cuda().to(BF).train()


def stepper(kind, model):
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    if kind == "module-mx":
        return ModuleStepper(model, info(), lr=1e-4, native=fused.NativeOptim())
    return FusedPythiaStepper(model, info(), lr=1e-4, quantize="mxfp8" if kind == "fused-mx" else None)


def frozen_bytes(kind, st):
    mods = list(st.model.relora_modules())
    if kind == "fused-bf16":
        return sum(m.weight.numel() * m.weight.element_size() for m in mods)
    return sum(m.frozen_weight_nbytes() for m in mods)


def train_rounds(name, T, steps, rounds):
    B = SHAPES[name][4]
    sts = {}
    packed = build(name, "mxfp8")
    models = {"fused-mx": packed, "module-mx": copy.deepcopy(packed)}  # the same packed bytes on both paths
    del packed
    for k in KINDS:
        gc.collect()
        torch.cuda.empty_cache()
        m0 = torch.cuda.memory_allocated()
        sts[k] = stepper(k, models.pop(k) if k in models else build(name, None))
        torch.cuda.synchronize()
        print(json.dumps({"shape": name, "executor": k, "frozen_weight_bytes": frozen_bytes(k, sts[k]),
                          "allocated_after_construction": torch.cuda.memory_allocated() - m0}), flush=True)
    ids = torch.randint(0, 50304, (B, T), generator=torch.Generator().manual_seed(1)).cuda()
    for k in KINDS:  # warm-up: graph capture, tensor maps, allocator
        for _ in range(2):
            sts[k].micro_step(ids)
            sts[k].update()
    torch.cuda.synchronize()
    rates = {k: [] for k in KINDS}
    for _ in range(rounds):
        for k in KINDS:  # the three executors alternate
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                loss = sts[k].micro_step(ids)
                sts[k].update()
            torch.cuda.synchronize()
            rates[k].append(B * T * steps / (time.perf_counter() - t0))
            assert torch.isfinite(loss), (k, float(loss))
    best = {k: max(v) for k, v in rates.items()}
    for k in KINDS:
        print(json.dumps({"shape": name, "executor": k, "tokens_per_s": [round(v) for v in sorted(rates[k])], "B": B, "T": T, "r": 128,
                          "dropout": 0.1, "best_vs_module_mx": round(best[k] / best["module-mx"], 2),
                          "best_vs_fused_bf16": round(best[k] / best["fused-bf16"], 2)}), flush=True)
    del sts
    gc.collect()
    torch.cuda.empty_cache()


def gemm_rows(name, T, P=None):
    """gemm_mx with its bias (packed weight K-major) against fused.gemm in bf16 with its bias, operands ready; the input gradient
    (the same bytes MN-major) against the bf16 GEMM's."""
    from relora_b200.ops import fused, mx

    C = fused._C()
    h, _, _, f, B = SHAPES[name]
    M = B * T
    flush = torch.empty(64 * 2**20, dtype=torch.float32, device="cuda")  # 256 MB, past the 50 MB L2
    for site, N, K in (("query_key_value", 3 * h, h), ("dense", h, h), ("dense_h_to_4h", f, h), ("dense_4h_to_h", h, f)):
        g = torch.Generator(device="cuda").manual_seed(N + K)
        x = torch.randn(M, K, generator=g, device="cuda").to(BF)
        w = (torch.randn(N, K, generator=g, device="cuda") * 0.02).to(BF)
        bias = (torch.randn(N, generator=g, device="cuda") * 0.02).to(BF)
        dy = torch.randn(M, N, generator=g, device="cuda").to(BF)
        mw, (xq, sfx), (dq, sfd) = mx.quantize_weight(w), mx.quantize_rows(x), mx.quantize_rows(dy)
        y, dx = torch.empty(M, N, dtype=BF, device="cuda"), torch.empty(M, K, dtype=BF, device="cuda")
        fl = 2.0 * M * N * K
        row = {}
        if P is not None:
            y0, y1 = torch.empty_like(y), torch.empty_like(y)
            C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y1, M, N, K, False)
            P.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y0, M, N, K, False, None, None, None)
            dx0, dx1 = torch.empty_like(dx), torch.empty_like(dx)
            C.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx1, M, K, N, True)
            P.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx0, M, K, N, True, None, None, None)
            torch.cuda.synchronize()
            row = {"parent_fwd_bit_identical": bool(torch.equal(y1.view(torch.int16), y0.view(torch.int16))),
                   "parent_dx_bit_identical": bool(torch.equal(dx1.view(torch.int16), dx0.view(torch.int16))),
                   "parent_mx_fwd_us": round(timeit(lambda: P.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y0, M, N, K, False, None, None, None),
                                                    flush), 1)}
        t = {
            "mx_fwd_bias": timeit(lambda: C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y, M, N, K, False, None, None, None, 0, 0, bias), flush),
            "mx_fwd": timeit(lambda: C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y, M, N, K, False), flush),
            "bf16_fwd_bias": timeit(lambda: fused.gemm(x, w, y, M=M, N=N, K1=K, bias=bias), flush),
            "mx_dx": timeit(lambda: C.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx, M, K, N, True), flush),
            "bf16_dx": timeit(lambda: fused.gemm(dy, w, dx, M=M, N=K, K1=N, b1_mn=True), flush),
        }
        print(json.dumps({"shape": name, "site": site, "M": M, "N": N, "K": K,
                          **{f"{k}_us": round(v, 1) for k, v in t.items()},
                          **{f"{k}_tflops": round(fl / v / 1e6, 1) for k, v in t.items()}, **row}), flush=True)
        del mw, xq, sfx, dq, sfd, x, w, dy, y, dx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["160m", "410m", "1b"])
    ap.add_argument("--train", nargs="*", default=None, help="shapes to train (default: --shapes)")
    ap.add_argument("--T", type=int, default=2049)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent-so", default=None)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    P = None
    if a.parent_so:
        import importlib.util

        spec = importlib.util.spec_from_file_location("parent_build._C", a.parent_so)
        P = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(P)
    for name in a.shapes:
        gemm_rows(name, a.T, P)
    for name in (a.shapes if a.train is None else a.train):
        train_rounds(name, a.T, a.steps, a.rounds)


if __name__ == "__main__":
    main()
