"""`--activation_checkpointing` on the fused executors: tokens/s and peak memory of save mode and recompute mode, alternating on one
card after warm-up.  Prints one JSON line per shape; the card's name and power limit are read in the same run.

    python bench/recompute_bench.py [--shapes llama_250m llama_1b pythia_1b llama31_8b] [--steps 4] [--rounds 2]

Random weights, ReLoRA r = 128, lora_dropout 0.1, CUDA graphs on:

* llama_250m, llama_1b: ``configs/*.json`` at ``bench.py``'s micro-batches (24 and 16 x 512 tokens);
* pythia_1b: ``bench/pythia_bench.py``'s 1B shape at T = 2049, one sequence;
* llama31_8b: Llama-3.1-8B's shape (h 4096, f 14336, 32 layers, 8 KV heads, 128,256-token vocabulary) at T = 8192, one sequence.
  Its head_dim of 128 runs SDPA (``--attention auto``).

A step is one micro-batch and one update.  ``peak_gb`` is ``torch.cuda.max_memory_allocated`` over a mode's warm-up, less what
was allocated before its model was built.  Recompute mode runs first; save mode is skipped, and the line says so, when its peak
predicted from the buffer shapes (recompute mode's peak plus L - 2 slots of every per-layer buffer) exceeds the free memory.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import torch  # noqa: E402

from pythia_bench import SHAPES as PYTHIA, gpu_info  # noqa: E402

BF = torch.bfloat16
GB = 1 << 30
# name: (builder, batch, T)
CASES = {
    "llama_250m": ("llama_250m", 24, 512),
    "llama_1b": ("llama_1b", 16, 512),
    "pythia_1b": ("pythia_1b", 1, 2049),
    "llama31_8b": ("llama31_8b", 1, 8192),
}


def info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def build(name):
    """The ReLoRA model of a case, built on the GPU in bf16."""
    from relora_b200.models import GPTNeoXForCausalLM, LlamaForCausalLM, SimpleConfig, load_config
    from relora_b200.relora import ReLoRaModel

    if name.startswith("pythia"):
        h, L, nh, f, _ = PYTHIA[name.split("_")[1]]
        cfg = SimpleConfig(model_type="gpt_neox", vocab_size=50304, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                           intermediate_size=f, rotary_pct=0.25, max_position_embeddings=2048, layer_norm_eps=1e-5,
                           use_parallel_residual=True, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
        cls, targets = GPTNeoXForCausalLM, ["attn", "attention", "mlp"]
    elif name == "llama31_8b":
        cfg = SimpleConfig(model_type="llama", vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                           num_attention_heads=32, num_key_value_heads=8, rms_norm_eps=1e-5, rope_theta=500000.0, pad_token_id=-1,
                           max_position_embeddings=8192)
        cls, targets = LlamaForCausalLM, ["attn", "mlp"]
    else:
        cfg = load_config(os.path.join(ROOT, "configs", f"{name}.json"))
        cls, targets = LlamaForCausalLM, ["attn", "mlp"]
    torch.manual_seed(0)
    dtype = torch.get_default_dtype()
    torch.set_default_dtype(BF)  # an 8B model in fp32 on the host would take 32 GB and minutes to initialise
    try:
        with torch.device("cuda"):
            w = ReLoRaModel(cls(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=targets, init_lora_a="kaiming")
    finally:
        torch.set_default_dtype(dtype)
    with torch.no_grad():
        for m in w.relora_modules():
            torch.nn.init.normal_(m.lora_B.weight, std=0.02)
    return w.cuda().to(BF).train(), cfg


def stepper(name, model, ckpt):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.fused_pythia import FusedPythiaStepper

    cls = FusedPythiaStepper if name.startswith("pythia") else FusedLlamaStepper
    return cls(model, info(), lr=1e-4, grad_accumulation=1, cuda_graphs=True, activation_checkpointing=ckpt)


def step(st, ids):
    st.micro_step(ids)
    st.update()


def warm(name, ckpt, ids, n):
    """Builds a mode's model and stepper and runs ``n`` steps; returns (stepper, peak bytes of the mode)."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    model, _ = build(name)
    st = stepper(name, model, ckpt)
    for _ in range(n):
        step(st, ids)
    torch.cuda.synchronize()
    return st, torch.cuda.max_memory_allocated() - before


def timed(st, ids, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        step(st, ids)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def run(name, args):
    _, B, T = CASES[name]
    V = 50304 if name.startswith("pythia") else (128256 if name == "llama31_8b" else 32100)
    ids = torch.randint(0, V, (B, T), generator=torch.Generator().manual_seed(0)).cuda()
    row = {"shape": name, "B": B, "T": T, "gpu": gpu_info()}
    rec, row["recompute_peak_gb"] = warm(name, True, ids, args.warmup)
    row["recompute_peak_gb"] /= GB
    L = rec.L
    per_layer = rec.saved_bytes_per_layer()
    predicted = row["recompute_peak_gb"] + (L - rec.n_slots) * per_layer / GB
    row["save_peak_predicted_gb"] = predicted
    free, total = torch.cuda.mem_get_info()
    avail = (free + torch.cuda.memory_reserved() - torch.cuda.memory_allocated()) / GB
    save = None
    if predicted > 0.95 * avail:
        # not next to the recompute stepper: would it fit on the card alone?
        row["save_skipped"] = (f"save mode is predicted to need {predicted:.1f} GB; {avail:.1f} GB are free next to recompute mode"
                               + (" and the card has " f"{total / GB:.1f} GB in all" if predicted > 0.95 * total / GB else ""))
    else:
        save, row["save_peak_gb"] = warm(name, False, ids, args.warmup)
        row["save_peak_gb"] /= GB
    tok = {"recompute": [], "save": []}
    for _ in range(args.rounds):
        for mode, st in (("save", save), ("recompute", rec)):
            if st is not None:
                tok[mode].append(B * T * args.steps / timed(st, ids, args.steps))
    for mode, v in tok.items():
        if v:
            row[f"{mode}_tokens_per_s"] = sorted(v)[len(v) // 2]
    if save is not None:
        row["recompute_vs_save_speed"] = row["recompute_tokens_per_s"] / row["save_tokens_per_s"]
        row["memory_saved_gb"] = row["save_peak_gb"] - row["recompute_peak_gb"]
    row["predicted_saving_gb"] = (L - rec.n_slots) * per_layer / GB
    del rec, save
    gc.collect()
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=list(CASES), choices=list(CASES))
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("recompute_bench.py needs a CUDA device")
    from relora_b200.ops import native

    native.require()
    for name in args.shapes:
        try:
            row = run(name, args)
        except torch.cuda.OutOfMemoryError as e:  # a prediction that was wrong: say so and go on with the next shape
            row = {"shape": name, "error": str(e)[:300]}
            gc.collect()
            torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
