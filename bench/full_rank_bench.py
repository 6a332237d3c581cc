"""Full-rank training: the fused executors against the module path, and the weight-gradient GEMM against cuBLAS.

    python bench/full_rank_bench.py [--models llama_250m,llama_1b] [--steps 8] [--rounds 3] [--out FILE]
    python bench/full_rank_bench.py --models pythia_160m,pythia_410m,pythia_1b [--ga 4]

Llama models come from ``configs/<name>.json`` (T 512).  Pythia models are GPT-NeoX at the shapes and batches of
``bench/pythia_bench.py`` (V 50304, parallel residual, rotary 0.25, GELU, T 2049, the recipe's sequence length); their rows also
carry an estimate of the fused executor's memory from shapes (bf16 parameters, fp32 gradients and AdamW moments, and the
activations the executor saves per token), printed next to the measured peak.

End to end: both executors train the same model from identical weights on the same seeded token batches, in one process.  After
a warm-up of both, they alternate ``--rounds`` times, each round timing ``--steps`` updates (``--ga`` micro-batches per update,
default 1) between device synchronises; the median tokens/s of each is reported, with the loss both reached after the same steps.
The fused executor's peak memory (``torch.cuda.max_memory_allocated``) is taken before the module path is built.

Per kernel: ``gW += dyᵀ·x`` (fp32, both operands MN-major) at the full-rank projection shapes of both models over 12 288 tokens,
split-K on (the default) and off (``--deterministic``), against ``torch.addmm(gW, dy.t(), x, out_dtype=torch.float32)``.  CUDA
events, 3 warm-up + 10 timed launches with a 256 MB write between launches to flush the L2, median.

The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from relora_b200.ops import fused as F  # noqa: E402

BF = torch.bfloat16
BATCH = {"llama_250m": 24, "llama_1b": 16}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


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


def wgrad_rows(cfg, name, M, flush):
    """dWqkv, dWo, dWgu, dWd of one layer: gW [N, K] += dy[M, N]ᵀ · x[M, K]."""
    h, fp = cfg.hidden_size, (cfg.intermediate_size + 127) // 128 * 128
    kv = getattr(cfg, "num_key_value_heads", None) or cfg.num_attention_heads
    kv = kv * (h // cfg.num_attention_heads)
    rows = []
    for site, N, K in (("dWqkv", h + 2 * kv, h), ("dWo", h, h), ("dWgu", 2 * fp, h), ("dWd", h, fp)):
        dy = torch.randn(M, N, device="cuda").to(BF)
        x = torch.randn(M, K, device="cuda").to(BF)
        gW = torch.zeros(N, K, device="cuda", dtype=torch.float32)
        flops = 2.0 * M * N * K
        rec = {"model": name, "site": site, "M": M, "N": N, "K": K}
        t = timeit(lambda: torch.addmm(gW, dy.t(), x, out_dtype=torch.float32), flush)
        rec.update(cublas_us=t * 1e6, cublas_tflops=flops / t / 1e12)
        for tag, sk in (("splitk", 0), ("deterministic", 1)):
            t = timeit(lambda: F.gemm(dy, x, gW, M=N, N=K, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=sk), flush)
            rec.update({f"ours_{tag}_us": t * 1e6, f"ours_{tag}_tflops": flops / t / 1e12})
        rows.append(rec)
        print(json.dumps(rec), flush=True)
    return rows


def pythia_config(name):
    from pythia_bench import SHAPES  # bench/ is on sys.path when this file runs as a script

    from relora_b200.models import SimpleConfig

    h, L, nh, f, B = SHAPES[name[len("pythia_"):]]
    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=50304, hidden_size=h, num_hidden_layers=L, num_attention_heads=nh,
                       intermediate_size=f, rotary_pct=0.25, max_position_embeddings=2048, layer_norm_eps=1e-5,
                       use_parallel_residual=True, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    return cfg, B


def pythia_memory_estimate(cfg, B, T, native_attn):
    """Bytes the fused full-rank executor holds, from shapes: 14 bytes per parameter (bf16 value, fp32 gradient, two fp32 AdamW
    moments), and per token and layer the bf16 tensors it saves for the backward (input, the two norm outputs, the post-rotary
    qkv, the attention output (twice with the wgmma kernels), the pre-GELU and GELU outputs; plus the sequential residual's x1)
    and the fp32 norm statistics.  Transients (one layer's gradients, the LM-head chunk) are not counted."""
    h, f, L, V = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers, cfg.vocab_size
    per_layer = 4 * h * h + 2 * h * f + 9 * h + f  # query_key_value + dense, the two MLP projections; biases and norms
    P = L * per_layer + 2 * V * h + 2 * h
    saved = 2 * ((1 + 2 + 3 + 1 + int(native_attn) + int(not cfg.use_parallel_residual)) * h + 2 * f) + 4 * 2 * (
        1 + int(not cfg.use_parallel_residual))
    per_token = L * saved + 2 * h  # and the last layer's output
    return {"params": P, "state_GB": 14 * P / 1e9, "saved_activations_per_token_MB": per_token / 1e6,
            "saved_activations_GB": per_token * B * T / 1e9, "total_GB": (14 * P + per_token * B * T) / 1e9}


def end_to_end(name, steps, rounds, warmup, T=512, ga=1):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.models import GPTNeoXForCausalLM, LlamaForCausalLM, load_config
    from relora_b200.parallel.dist import DistInfo

    info = DistInfo(0, 0, 1, torch.device("cuda", torch.cuda.current_device()), "nccl")
    pythia = name.startswith("pythia_")
    if pythia:
        cfg, B = pythia_config(name)
        T = 2049
    else:
        cfg = load_config(os.path.join(ROOT, "configs", f"{name}.json"))
        B = BATCH[name]
    Fused = FusedPythiaStepper if pythia else FusedLlamaStepper
    torch.manual_seed(0)
    host = (GPTNeoXForCausalLM if pythia else LlamaForCausalLM)(cfg).to(BF)
    g = torch.Generator().manual_seed(1)
    n_total = warmup + steps * rounds
    batches = [torch.randint(0, cfg.vocab_size, (B, T), generator=g) for _ in range(n_total * ga)]
    kw = dict(lr=3e-4, weight_decay=0.0, clip_grad_norm=1.0, grad_accumulation=ga)

    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    st = {"fused": Fused(copy.deepcopy(host).cuda(), info, cuda_graphs=True, **kw)}
    pos = {"fused": 0, "module": 0}
    losses = {"fused": [], "module": []}

    def run(eng, n):
        s = st[eng]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            for _ in range(ga):
                ids = batches[pos[eng]].cuda(non_blocking=True)
                losses[eng].append(s.micro_step(ids))
                pos[eng] += 1
            s.update()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    run("fused", warmup)
    fused_peak = torch.cuda.max_memory_allocated()
    st["module"] = ModuleStepper(copy.deepcopy(host).cuda(), info, native=F.NativeOptim(), **kw)
    del host
    run("module", warmup)
    tps = {"fused": [], "module": []}
    for _ in range(rounds):
        for eng in ("fused", "module"):
            tps[eng].append(steps * ga * B * T / run(eng, steps))
    med = {k: sorted(v)[len(v) // 2] for k, v in tps.items()}
    rec = {"model": name, "batch": B, "seq": T, "grad_accumulation": ga, "steps_per_round": steps, "rounds": rounds,
           "fused_tokens_per_s": med["fused"], "module_tokens_per_s": med["module"], "fused_over_module": med["fused"] / med["module"],
           "fused_tokens_per_s_all": tps["fused"], "module_tokens_per_s_all": tps["module"],
           "final_loss_fused": float(losses["fused"][-1]), "final_loss_module": float(losses["module"][-1]), "after_updates": n_total,
           "fused_max_memory_allocated_GB": fused_peak / 1e9}
    if pythia:
        rec["fused_memory_estimate"] = pythia_memory_estimate(cfg, B, T, st["fused"].native_attn)  # per micro-batch
        rec["attention_native"] = st["fused"].native_attn
    print(json.dumps(rec), flush=True)
    del st
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama_250m,llama_1b")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ga", type=int, default=1, help="micro-batches per update (gradient accumulation)")
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("full_rank_bench needs a CUDA device")
    from relora_b200.models import load_config

    names = a.models.split(",")
    res = {"card": card(), "wgrad": [], "e2e": []}
    print(json.dumps(res["card"]), flush=True)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    for name in (n for n in names if not n.startswith("pythia_")):  # the dW GEMM rows cover the Llama configs
        res["wgrad"] += wgrad_rows(load_config(os.path.join(ROOT, "configs", f"{name}.json")), name, 12288, flush)
    del flush
    if not a.skip_e2e:
        for name in names:
            res["e2e"].append(end_to_end(name, a.steps, a.rounds, a.warmup, ga=a.ga))
    res["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
