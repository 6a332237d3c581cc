"""Llama-3 vocabularies on one GPU: the cross-entropy kernel at 32K, 50K and 128K tokens, and ReLoRA training tokens/s of a
Llama-3.1-8B-shaped model, fused executor vs module path.

    python bench/llama3_bench.py [--layers 2] [--steps 5] [--warmup 2] [--out llama3_bench.json] [--skip-model]

Kernel rows: ``cross_entropy_fwd_bwd`` on M = 4096 rows of bf16 logits, V in {32000, 50304, 128256} (the last one takes the
streaming kernel, the others the single-pass kernel that stages a row in shared memory); CUDA events, L2 flushed between launches,
the median of 20.  ``bytes`` is what any kernel must move, each logit read once and its gradient written once (2 x 2 bytes per
element); ``share_of_hbm_bound`` is that over 3.35 TB/s (H100 SXM data sheet) against the measured time.  The streaming kernel
reads each row three times, so its own traffic is up to twice ``bytes``, less what passes 2 and 3 find in L2.

Model row: h 4096, 32 query heads, 8 KV heads, intermediate 14336, vocab 128256, llama3 RoPE (factor 8, low/high frequency
factors 1 and 4, 8192 original positions, θ 500000), untied embeddings, T 2048, batch 1, ReLoRA r 128, lora_dropout 0.1, random
weights, ``--layers`` decoder layers (32 in the real model).  Both paths start from the same weights; after warm-up of both they
alternate, each step (micro-step + update) timed with CUDA events.  The loss and the worst gradient relative error of fused vs
module come from one micro-step on identical weights and dropout masks.  The card name, power limit and maximum SM clock
(read-only nvidia-smi query) are recorded with the rows."""
from __future__ import annotations

import argparse
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

import torch  # noqa: E402

from gqa_bench import timeit  # noqa: E402
from pythia_bench import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def ce_rows(C, M=4096):
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for V in (32000, 50304, 128256):
        ldv = (V + 7) // 8 * 8
        logits = (torch.randn(M, ldv, device="cuda", generator=g) * 2.0).bfloat16()
        labels = torch.randint(0, V, (M,), device="cuda", generator=g)
        loss_sum = torch.zeros(1, device="cuda")
        count = torch.zeros(1, device="cuda")
        # in place: later launches see the gradients of earlier ones, which costs the kernel the same
        t = timeit(lambda: C.cross_entropy_fwd_bwd(logits, labels, V, 1.0, -100, loss_sum, count), flush, iters=20)
        nbytes = 2 * 2 * M * V + 8 * M
        row = {"M": M, "V": V, "kernel": "ce_stream_kernel" if V * 2 > 200 * 1024 else "ce_kernel", "us": t, "bytes": nbytes,
               "gb_per_s": nbytes / t / 1e3, "share_of_hbm_bound": nbytes / HBM_BYTES_PER_S * 1e6 / t}
        print(json.dumps({k: (round(x, 3) if isinstance(x, float) else x) for k, x in row.items()}), flush=True)
        rows.append(row)
        del logits
    return rows


def model_row(layers, steps, warmup):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.ops import fused
    from relora_b200.parallel.dist import DistInfo
    from relora_b200.relora import ReLoRaModel

    dev = torch.device("cuda", 0)
    info = DistInfo(0, 0, 1, dev, "nccl")
    h, nh, nkv, f, V, T, B = 4096, 32, 8, 14336, 128256, 2048, 1
    rope = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}
    cfg = SimpleConfig(model_type="llama", vocab_size=V, hidden_size=h, intermediate_size=f, num_hidden_layers=layers,
                       num_attention_heads=nh, num_key_value_heads=nkv, rms_norm_eps=1e-5, max_position_embeddings=131072,
                       rope_theta=500000.0, rope_scaling=rope, tie_word_embeddings=False)
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
    for st in steppers.values():
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
    row = {"shape": "llama3.1_8b", "hidden": h, "layers": layers, "heads": nh, "kv_heads": nkv, "intermediate": f, "vocab": V,
           "T": T, "batch": B, "tokens_per_s_fused": tok / times["fused"], "tokens_per_s_module": tok / times["module"],
           "speedup": times["module"] / times["fused"], "loss_fused": lf, "loss_module": lm, "worst_grad_relerr": worst,
           "worst_grad_param": worst_name, "attention_native": fs.native_attn,
           "peak_memory_gb": torch.cuda.max_memory_allocated() / 2**30}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=2, help="decoder layers of the model row (32 in Llama-3.1-8B)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="llama3_bench.json", help="where the JSON result goes")
    ap.add_argument("--skip-model", action="store_true", help="only the cross-entropy rows")
    a = ap.parse_args()
    from relora_b200.ops import native

    C = native.require()
    res = {"gpu": gpu_info(), "cross_entropy": ce_rows(C)}
    if not a.skip_model:
        res["model"] = model_row(a.layers, a.steps, a.warmup)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
