"""Tokens/s of the Pythia fused executor (--engine fused) vs the module path (--engine module) on one GPU, in one process.

    python bench/pythia_bench.py [--steps 10] [--warmup 3] [--out pythia_bench.json] [--shapes 160m,410m,1b]

Random weights; ReLoRA r = 128, lora_dropout 0.1, T = 2049 (the 1B recipe's sequence length), rotary 0.25, parallel residual.  Both
paths are built from the same weights; every shape is warmed up on both before timing, then the two paths alternate, each timed
window measured with CUDA events.  At each shape the loss and the worst gradient relative error of fused vs module (one micro-step on
identical weights and dropout masks) are recorded with the card name, power limit and maximum SM clock."""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SHAPES = {  # name: (hidden, layers, heads, intermediate, batch)
    "160m": (768, 12, 12, 3072, 4),
    "410m": (1024, 24, 16, 4096, 2),
    "1b": (2048, 16, 8, 8192, 1),
}


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
        name, power, clock = [s.strip() for s in out.splitlines()[0].split(",")]
    except Exception:
        name, power, clock = torch.cuda.get_device_name(0), "unknown", "unknown"
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def build_model(h, L, nh, f, seed=0):
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=50304, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                       intermediate_size=f, rotary_pct=0.25, max_position_embeddings=2048, layer_norm_eps=1e-5,
                       use_parallel_residual=True, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    torch.manual_seed(seed)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming")
    with torch.no_grad():
        for m in w.relora_modules():
            torch.nn.init.normal_(m.lora_B.weight, std=0.02)
    return w.cuda().to(torch.bfloat16).train()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--T", type=int, default=2049)
    ap.add_argument("--shapes", default="160m,410m,1b")
    ap.add_argument("--out", default="pythia_bench.json", help="where the JSON result goes")
    a = ap.parse_args()
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused
    from relora_b200.parallel.dist import DistInfo

    dev = torch.device("cuda", 0)
    info = DistInfo(0, 0, 1, dev, "nccl")
    res = {"gpu": gpu_info(), "T": a.T, "steps": a.steps, "warmup": a.warmup, "rows": []}
    for name in a.shapes.split(","):
        h, L, nh, f, B = SHAPES[name]
        wa = build_model(h, L, nh, f)
        wb = copy.deepcopy(wa)
        fs = FusedPythiaStepper(wa, info, lr=1e-4, cuda_graphs=True)
        ms = ModuleStepper(wb, info, lr=1e-4, native=fused.NativeOptim())
        g = torch.Generator(device=dev).manual_seed(1)
        ids = torch.randint(0, 50304, (B, a.T), device=dev, generator=g)
        # outputs on identical weights and masks (before any update)
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
            for _ in range(a.warmup):
                st.micro_step(ids)
                st.update()
        torch.cuda.synchronize()
        times = {k: 0.0 for k in steppers}
        for _ in range(a.steps):
            for k, st in steppers.items():  # alternate the two paths
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                st.micro_step(ids)
                st.update()
                e1.record()
                e1.synchronize()
                times[k] += e0.elapsed_time(e1) / 1e3
        tok = B * a.T * a.steps
        row = {"shape": name, "hidden": h, "layers": L, "heads": nh, "head_dim": h // nh, "intermediate": f, "batch": B,
               "tokens_per_s_fused": tok / times["fused"], "tokens_per_s_module": tok / times["module"],
               "speedup": times["module"] / times["fused"], "loss_fused": lf, "loss_module": lm,
               "worst_grad_relerr": worst, "worst_grad_param": worst_name, "attention_native": fs.native_attn}
        print(json.dumps(row), flush=True)
        res["rows"].append(row)
        del fs, ms, wa, wb, steppers
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
