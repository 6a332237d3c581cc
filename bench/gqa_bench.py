"""Grouped-query attention on one GPU: the wgmma GQA kernels vs torch SDPA (``enable_gqa``), and ReLoRA training tokens/s of a
GQA Llama at the TinyLlama-1.1B shape, fused executor vs module path.

    python bench/gqa_bench.py [--steps 5] [--warmup 2] [--out gqa_bench.json] [--skip-model]

Kernel rows: B 4, T 2048, 32 query heads, head_dim 64 and 128, group sizes (query heads per KV head) 4 and 8; CUDA events, L2
flushed between launches, the median of 10.  FLOPs count the causal half of the score matrix.

Model row: the fused executor vs the module path (``--engine fused`` / ``--engine module``) at the TinyLlama-1.1B shape: h 2048,
22 layers, 32 query heads, 4 KV heads, intermediate 5632, vocab 32000, T 2048, batch 1, ReLoRA r 128, lora_dropout 0.1, random
weights, default ``--attention auto``.  Both paths start from the same weights; after warm-up of both they alternate, each step
timed with CUDA events.  The loss and the worst gradient relative error of fused vs module come from one micro-step on identical
weights and dropout masks.  The card name, power limit and
maximum SM clock (read-only nvidia-smi query) are recorded with the rows."""
from __future__ import annotations

import argparse
import copy
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

import torch  # noqa: E402
import torch.nn.functional as Fn  # noqa: E402

from pythia_bench import gpu_info  # noqa: E402


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
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def kernel_rows(C):
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    rows = []
    B, T, nh = 4, 2048, 32
    for hd in (64, 128):
        for group in (4, 8):
            nkv = nh // group
            qkv = (torch.randn(B * T, (nh + 2 * nkv) * hd, device="cuda") * 0.5).bfloat16()
            out = torch.empty(B * T, nh * hd, device="cuda", dtype=torch.bfloat16)
            lse = torch.empty(B, nh, T, device="cuda", dtype=torch.float32)
            delta = torch.empty_like(lse)
            dout = (torch.randn(B * T, nh * hd, device="cuda") * 0.1).bfloat16()
            dqkv = torch.empty_like(qkv)
            sc = 1.0 / math.sqrt(hd)
            t_f = timeit(lambda: C.attention_fwd(qkv, out, lse, B, T, nh, hd, sc, nkv=nkv), flush)
            t_b = timeit(lambda: C.attention_bwd(qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, sc, nkv=nkv), flush)
            v3 = qkv.view(B, T, nh + 2 * nkv, hd).transpose(1, 2)
            q, k, v = (t.detach().requires_grad_() for t in (v3[:, :nh], v3[:, nh:nh + nkv], v3[:, nh + nkv:]))
            sdpa = lambda: Fn.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True)  # noqa: E731
            t_sf = timeit(sdpa, flush)
            o = sdpa()
            g = dout.view(B, T, nh, hd).transpose(1, 2)
            t_sb = timeit(lambda: torch.autograd.grad(o, (q, k, v), g, retain_graph=True), flush)
            fl = 4.0 * B * nh * T * T * hd / 2
            row = {"B": B, "T": T, "nh": nh, "nkv": nkv, "group": group, "hd": hd, "ours_fwd_us": t_f, "sdpa_fwd_us": t_sf,
                   "ours_bwd_us": t_b, "sdpa_bwd_us": t_sb, "ours_fwd_tflops": fl / t_f / 1e6, "ours_bwd_tflops": 2.5 * fl / t_b / 1e6}
            print(json.dumps({k_: (round(x, 1) if isinstance(x, float) else x) for k_, x in row.items()}), flush=True)
            rows.append(row)
    return rows


def model_row(steps, warmup):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.ops import fused
    from relora_b200.parallel.dist import DistInfo
    from relora_b200.relora import ReLoRaModel

    dev = torch.device("cuda", 0)
    info = DistInfo(0, 0, 1, dev, "nccl")
    h, L, nh, nkv, f, V, T, B = 2048, 22, 32, 4, 5632, 32000, 2048, 1
    cfg = SimpleConfig(model_type="llama", vocab_size=V, hidden_size=h, intermediate_size=f, num_hidden_layers=L,
                       num_attention_heads=nh, num_key_value_heads=nkv, rms_norm_eps=1e-5, max_position_embeddings=T)
    torch.manual_seed(0)
    wa = ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "mlp"], init_lora_a="kaiming")
    with torch.no_grad():
        for m in wa.relora_modules():
            torch.nn.init.normal_(m.lora_B.weight, std=0.02)
    wa = wa.cuda().to(torch.bfloat16).train()
    wb = copy.deepcopy(wa)
    fs = FusedLlamaStepper(wa, info, lr=1e-4, cuda_graphs=True)
    ms = ModuleStepper(wb, info, lr=1e-4, native=fused.NativeOptim())
    ids = torch.randint(0, V, (B, T), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    # outputs on identical weights and dropout masks (before any update)
    fused.seed_state.set(dev, 11)
    lf = float(fs.micro_step(ids))
    fused.seed_state.set(dev, 11)
    lm = float(ms.micro_step(ids))
    worst, worst_name = 0.0, ""
    mod = dict(zip(ms.trainable_names, ms.trainable_params))
    for n, p in zip(fs.trainable_names, fs.trainable_params):
        gf, gm = fs.store.view_like(fs.store.grads, p).float(), ms.store.view_like(ms.store.grads, mod[n]).float()
        if gm.norm() > 0:
            e = float((gf - gm).norm() / gm.norm())
            if e > worst:
                worst, worst_name = e, n
    fs.optimizer.zero_grad()
    ms.optimizer.zero_grad()
    steppers = {"fused": fs, "module": ms}
    for st in steppers.values():  # warm-up: graph capture, allocator, library algorithm choice
        for _ in range(warmup):
            st.micro_step(ids)
            st.update()
    torch.cuda.synchronize()
    times = {k: 0.0 for k in steppers}
    for _ in range(steps):
        for k, st in steppers.items():  # alternate the two paths
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            st.micro_step(ids)
            st.update()
            e1.record()
            e1.synchronize()
            times[k] += e0.elapsed_time(e1) / 1e3
    tok = B * T * steps
    row = {"shape": "tinyllama_1.1b", "hidden": h, "layers": L, "heads": nh, "kv_heads": nkv, "intermediate": f, "vocab": V, "T": T,
           "batch": B, "tokens_per_s_fused": tok / times["fused"], "tokens_per_s_module": tok / times["module"],
           "speedup": times["module"] / times["fused"], "loss_fused": lf, "loss_module": lm, "worst_grad_relerr": worst,
           "worst_grad_param": worst_name, "attention_native": fs.native_attn}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="gqa_bench.json", help="where the JSON result goes")
    ap.add_argument("--skip-model", action="store_true", help="only the kernel rows")
    a = ap.parse_args()
    from relora_b200.ops import native

    C = native.require()
    res = {"gpu": gpu_info(), "kernels": kernel_rows(C)}
    if not a.skip_model:
        res["model"] = model_row(a.steps, a.warmup)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
