"""Bisect a non-finite multi-GPU training state (round-1 driver run: `last_loss = NaN` at N = 4 and 8 for this engine and a
`clip_grad_norm_` failure for the reference arm, both finite at N <= 2).

    python bench/nan_hunt.py drive --gpus 4 --steps 50          # runs the arms below one after another, decides what to run next
    torchrun ... bench/nan_hunt.py ours|ref|nccl --steps 50 --tag NAME

Every rank writes one JSON line per step to gpurun_out/nan_hunt/<tag>_rank<r>.jsonl:

* ours : this rank's loss before the cross-rank mean, the all-reduced [mean, skip], non-finite counts of the local fp32
         gradients (before the update), of the parameters and Adam moments (after it), the gradient norm returned by the
         fused update and a parameter checksum (replica equality);
* ref  : per-micro-batch losses, the first parameter whose (already all-reduced) gradient is non-finite, the clip norm;
* nccl : all-reduce stress (25 MB bf16 AVG buckets like DDP's, 3-float SUM like loss_info) against locally computed sums.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("RELORA_B200_NO_WANDB", "1")
os.environ.setdefault("WANDB_MODE", "disabled")
OUT = os.path.join(ROOT, "gpurun_out", "nan_hunt")


def _writer(tag, rank):
    os.makedirs(OUT, exist_ok=True)
    f = open(os.path.join(OUT, f"{tag}_rank{rank}.jsonl"), "w")

    def w(rec):
        f.write(json.dumps(rec) + "\n")
        f.flush()

    return w


def _setup():
    import torch
    import torch.distributed as dist

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return rank, world, local


def run_ours(a):
    import torch
    import torch.distributed as dist

    import bench as B
    from relora_b200.engine.api import TrainingEngine
    from relora_b200.models import load_config
    from relora_b200.parallel.dist import init_distributed

    rank, world, local = _setup()
    info = init_distributed("cuda", "nccl")
    w = _writer(a.tag, rank)
    if a.sdpa_backend != "default":  # which library kernel torch SDPA may pick (by default cuDNN's)
        torch.backends.cuda.enable_cudnn_sdp(a.sdpa_backend == "cudnn")
        torch.backends.cuda.enable_flash_sdp(a.sdpa_backend == "flash")
        torch.backends.cuda.enable_mem_efficient_sdp(a.sdpa_backend == "efficient")
        torch.backends.cuda.enable_math_sdp(a.sdpa_backend == "math")
    cfg_path = os.path.join(ROOT, "configs", f"{a.model}.json")
    rec = B.RECIPES[a.model]
    batch, ga = rec["batch"], a.ga or rec["ga"]
    eng = TrainingEngine.build(
        info, model_config=cfg_path, batch_size=batch, gradient_accumulation=ga, total_batch_size=batch * ga * world,
        max_length=512, use_peft=True, lora_r=128, relora=5000, cycle_length=5000, scheduler="cosine_restarts", warmup_steps=500,
        restart_warmup_steps=100, lr=1e-3, num_training_steps=20000, dtype="bfloat16", device="cuda", comm=a.comm,
        cuda_graphs=a.cuda_graphs == "true", attention=a.attention, **rec["reset"])
    vocab = load_config(cfg_path).vocab_size
    # the driver's data: seed 1234 + rank; --emulate_world W feeds rank r the concatenated micro-batches of W ranks (one GPU)
    if a.emulate_world > 1:
        host = torch.cat([B.make_tokens(a.steps, rec["ga"], batch, 512, vocab, r, pinned=False) for r in range(a.emulate_world)], dim=1)
    else:
        host = B.make_tokens(a.steps, ga, batch, 512, vocab, rank, pinned=False)
    toks = host.cuda()
    st = eng.stepper
    nf = lambda t: int((~torch.isfinite(t.float())).sum())  # noqa: E731
    first_bad = None
    for s in range(a.steps):
        total = None
        micro = []
        if s == a.pinpoint_step:
            _pinpoint(st, toks[s], w)
            break
        for i in range(toks.shape[1]):
            loss = st.micro_step(toks[s, i]).float()
            micro.append(loss)
            total = loss if total is None else total + loss
        local_mean = total / toks.shape[1]
        g_bad = nf(st.store.grads)
        g_abs = float(st.store.grads.float().abs().max())
        skip = torch.isnan(local_mean).float()
        pack = torch.stack([local_mean, skip])
        if world > 1:
            dist.all_reduce(pack)
        mean, skip = pack[0] / world, pack[1]
        upd = st.update(skip=skip)
        eng.optimizer._opt_called = True
        eng.scheduler.step()
        eng.update_step += 1
        p = st.store.params
        rec_ = {"step": s, "local_loss": float(local_mean), "micro": [float(x) for x in micro], "mean_loss": float(mean), "skip": float(skip),
                "grad_nonfinite": g_bad, "grad_absmax": g_abs, "grad_norm": float(upd.grad_norm), "param_nonfinite": nf(p),
                "m_nonfinite": nf(eng.optimizer.exp_avg), "v_nonfinite": nf(eng.optimizer.exp_avg_sq),
                "param_checksum": float(p.double().abs().sum()), "lr": eng.optimizer.param_groups[0]["lr"]}
        w(rec_)
        bad = (rec_["grad_nonfinite"] or rec_["param_nonfinite"] or rec_["local_loss"] != rec_["local_loss"]
               or rec_["grad_norm"] != rec_["grad_norm"] or rec_["mean_loss"] != rec_["mean_loss"])
        if bad and first_bad is None:
            first_bad = s
    res = {"tag": a.tag, "rank": rank, "first_bad_step": first_bad, "transport": getattr(st.sync, "transport", "none"),
           "multicast": os.environ.get("RELORA_B200_MULTICAST", "1")}
    w({"summary": res})
    flag = torch.tensor([-1 if first_bad is None else first_bad], device="cuda")
    gathered = [torch.zeros_like(flag) for _ in range(world)]
    dist.all_gather(gathered, flag)
    if rank == 0:
        print("RESULT " + json.dumps({"tag": a.tag, "first_bad_step_per_rank": [int(x) for x in gathered]}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


def _pinpoint(st, toks, w):
    """Re-run the micro-batches of one update without the CUDA graph / side stream, checking every kernel call's tensor arguments
    for non-finite values before and after the call.  The first call that turns clean arguments into non-finite ones is the
    culprit; its arguments (sliced to the offending batch element for attention) are saved to gpurun_out/nan_hunt/culprit.pt."""
    import torch

    from relora_b200.ops import fused

    found = {}

    def nonfinite(t):
        return int((~torch.isfinite(t.float())).sum()) if torch.is_tensor(t) and t.is_floating_point() and t.numel() else 0

    def tensors(args, kwargs):
        out = []
        for x in list(args) + list(kwargs.values()):
            if torch.is_tensor(x):
                out.append(x)
            elif isinstance(x, (list, tuple)):
                out += [y for y in x if torch.is_tensor(y)]
        return out

    def wrap(name, fn):
        def inner(*args, **kwargs):
            if found:
                return fn(*args, **kwargs)
            ts = tensors(args, kwargs)
            before = [nonfinite(t) for t in ts]
            res = fn(*args, **kwargs)
            outs = ts + tensors(res if isinstance(res, (list, tuple)) else [res], {})
            after = [nonfinite(t) for t in outs]
            if sum(before) == 0 and sum(after) > 0:
                found.update(name=name, after=after, shapes=[tuple(t.shape) for t in outs], dtypes=[str(t.dtype) for t in outs],
                             micro=state["micro"], call_index=state["calls"])
                found["tensors"] = [t.detach().clone() for t in outs]
            state["calls"] += 1
            return res
        return inner

    class Proxy:
        def __init__(self, real):
            self._real = real

        def __getattr__(self, k):
            v = getattr(self._real, k)
            return wrap("C." + k, v) if callable(v) else v

    state = {"micro": 0, "calls": 0}
    # phase 1 (fast, captured graph): which micro-batch turns the accumulated gradients non-finite?
    bad_i = None
    for i in range(toks.shape[0]):
        loss = st.micro_step(toks[i])
        nfg = nonfinite(st.store.grads)
        w({"scan_micro": i, "loss": float(loss), "grad_nonfinite": nfg})
        if nfg:
            bad_i = i
            break
    if bad_i is None:
        w({"culprit": None, "note": "no micro-batch of this update produced non-finite gradients"})
        return
    # phase 2: replay that micro-batch eagerly (no graph, no side stream) with every kernel call checked
    st.store.grads.zero_()
    st.use_graphs, st.side = False, None
    real_C, real_gemm, real_grad = st.C, fused.gemm, torch.autograd.grad
    st.C = Proxy(real_C)
    fused.gemm = wrap("gemm", real_gemm)
    torch.autograd.grad = wrap("sdpa_backward(autograd.grad)", real_grad)
    try:
        state["micro"], state["calls"] = bad_i, 0
        loss = st.micro_step(toks[bad_i])
        w({"pinpoint_micro": bad_i, "loss": float(loss), "grad_nonfinite": nonfinite(st.store.grads), "culprit": found.get("name")})
    finally:
        st.C, fused.gemm, torch.autograd.grad = real_C, real_gemm, real_grad
    if found:
        ts = found.pop("tensors")
        w({"culprit": found})
        # attention backward: outputs are (dq, dk, dv) after the inputs (o, (q, k, v), dO); keep the offending batch element only
        save = {}
        if found["name"].startswith("sdpa"):
            bad_b = None
            for t in ts:
                if t.dim() == 4 and nonfinite(t):
                    bad_b = int((~torch.isfinite(t.float())).flatten(1).any(1).nonzero()[0])
                    break
            for j, t in enumerate(ts):
                save[f"t{j}"] = (t[bad_b:bad_b + 1] if (t.dim() == 4 and bad_b is not None) else t).cpu()
            save["bad_batch"] = bad_b
        else:
            for j, t in enumerate(ts):
                if t.numel() * t.element_size() < 8e6:
                    save[f"t{j}"] = t.cpu()
        save["meta"] = found
        torch.save(save, os.path.join(OUT, "culprit.pt"))
    else:
        w({"culprit": None})


def run_ref(a):
    import torch
    import torch.distributed as dist

    import bench as B

    rank, world, local = _setup()
    w = _writer(a.tag, rank)
    B._stub_missing_modules()
    sys.path.insert(0, os.path.join(ROOT, "baseline", "_ref"))
    from peft_pretraining import training_utils
    from peft_pretraining.modeling_llama import LlamaForCausalLM
    from peft_pretraining.relora import ReLoRaModel
    from transformers import AutoConfig

    torch.manual_seed(0)
    device = f"cuda:{local}"
    rec = B.RECIPES[a.model]
    batch, ga = rec["batch"], rec["ga"]
    cfg = AutoConfig.from_pretrained(os.path.join(ROOT, "configs", f"{a.model}.json"))
    model = LlamaForCausalLM(cfg)
    model = ReLoRaModel(model, r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "attention", "mlp"], trainable_scaling=False,
                        keep_original_weights=True, lora_only=False, quantize=None, use_double_quant=True)
    model = model.to(device=device, dtype=torch.bfloat16)
    model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], output_device=local)
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    trainable = [p for _, p in named]
    optimizer = torch.optim.AdamW(trainable, lr=1e-3, weight_decay=0.0, betas=(0.9, 0.999))
    scheduler = training_utils.get_scheculer(optimizer=optimizer, scheduler_type="cosine_restarts", num_training_steps=20000, warmup_steps=500,
                                             min_lr_ratio=0.1, cycle_length=5000, restart_warmup_steps=100, adjust_step=0)
    toks = B.make_tokens(a.steps, ga, batch, 512, cfg.vocab_size, rank, pinned=False).to(device)
    first_bad = None
    for s in range(a.steps):
        micro = []
        for mb in range(ga):
            ids = toks[s, mb]
            loss = model(input_ids=ids, labels=ids).loss
            micro.append(float(loss))
            (loss / ga).backward()
        bad_names = [n for n, p in named if p.grad is not None and not bool(torch.isfinite(p.grad).all())]
        try:
            gn = float(torch.nn.utils.clip_grad_norm_(trainable, 1.0, error_if_nonfinite=True))
            err = None
        except RuntimeError as e:
            gn, err = float("nan"), str(e)[:200]
        p_bad = [n for n, p in named if not bool(torch.isfinite(p).all())]
        w({"step": s, "micro": micro, "grad_norm": gn, "bad_grads": bad_names[:8], "n_bad_grads": len(bad_names), "bad_params": p_bad[:8],
           "error": err, "lr": optimizer.param_groups[0]["lr"]})
        if err is not None or any(m != m for m in micro):
            first_bad = s
            break
        optimizer.step()
        scheduler.step()
        optimizer.zero_grad()
    flag = torch.tensor([-1 if first_bad is None else first_bad], device="cuda")
    gathered = [torch.zeros_like(flag) for _ in range(world)]
    dist.all_gather(gathered, flag)
    if rank == 0:
        print("RESULT " + json.dumps({"tag": a.tag, "first_bad_step_per_rank": [int(x) for x in gathered],
                                      "nvls_env": os.environ.get("NCCL_NVLS_ENABLE", "default")}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


def run_nccl(a):
    import torch
    import torch.distributed as dist

    rank, world, local = _setup()
    w = _writer(a.tag, rank)
    n = 12_500_000 // (8 * world) * 8 * world
    gens = [torch.Generator(device="cuda").manual_seed(77 + r) for r in range(world)]
    xs = [(torch.randn(n, device="cuda", generator=g) * 0.02).to(torch.bfloat16) for g in gens]
    expect = torch.stack([x.float() for x in xs]).mean(0)
    mine = xs[rank]
    bad_big = torch.zeros(1, device="cuda")
    worst = torch.zeros(1, device="cuda")
    buf = torch.empty_like(mine)
    for it in range(a.iters):
        buf.copy_(mine)
        dist.all_reduce(buf, op=dist.ReduceOp.AVG)
        err = (buf.float() - expect).abs()
        bad_big += (~torch.isfinite(buf.float())).sum() + (err > 2e-3).sum()
        worst = torch.maximum(worst, torch.nan_to_num(err.max(), nan=1e9).reshape(1))
    small_bad = torch.zeros(1, device="cuda")
    for it in range(a.iters * 2):
        t = torch.tensor([10.5 + rank, 1.0, 0.0], device="cuda")
        dist.all_reduce(t)
        want = torch.tensor([10.5 * world + world * (world - 1) / 2, float(world), 0.0], device="cuda")
        small_bad += (t != want).sum()
    res = {"tag": a.tag, "rank": rank, "bf16_avg_bad_elems": float(bad_big), "bf16_avg_worst_err": float(worst), "small_sum_bad": float(small_bad),
           "iters": a.iters, "nvls_env": os.environ.get("NCCL_NVLS_ENABLE", "default")}
    w(res)
    allr = [None] * world
    dist.all_gather_object(allr, res)
    if rank == 0:
        print("RESULT " + json.dumps({"tag": a.tag, "per_rank": allr}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


def drive(a):
    """Run the arms in order; later arms depend on what earlier ones showed.  Everything lands in gpurun_out/nan_hunt/."""
    os.makedirs(OUT, exist_ok=True)
    port = [29700]
    summary = {}

    def launch(mode, tag, extra_env=None, extra_args=(), timeout=600):
        port[0] += 2
        env = dict(os.environ, PYTHONPATH=ROOT, **(extra_env or {}))
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={a.gpus}", "--master-addr", "127.0.0.1",
               "--master-port", str(port[0]), os.path.abspath(__file__), mode, "--tag", tag, "--steps", str(a.steps), "--iters", str(a.iters),
               "--model", a.model, *extra_args]
        t0 = time.time()
        try:
            out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=timeout)
            rc, so, se = out.returncode, out.stdout, out.stderr
        except subprocess.TimeoutExpired as e:
            rc, so, se = -9, (e.stdout or b"").decode(errors="replace") if isinstance(e.stdout, bytes) else (e.stdout or ""), "TIMEOUT"
        with open(os.path.join(OUT, f"{tag}.log"), "w") as f:
            f.write(so + "\n=== stderr ===\n" + se[-20000:])
        res = None
        for line in so.splitlines():
            if line.startswith("RESULT "):
                res = json.loads(line[7:])
        summary[tag] = {"rc": rc, "seconds": round(time.time() - t0, 1), "result": res}
        with open(os.path.join(OUT, "summary.json"), "w") as f:
            json.dump(summary, f, indent=1)
        print(f"[hunt] {tag}: rc={rc} {summary[tag]['seconds']}s {res}", flush=True)
        return res

    def bad(res):
        return res is None or any(x >= 0 for x in res.get("first_bad_step_per_rank", [0]))

    r = launch("ours", "ours_default")
    if bad(r):
        r2 = launch("ours", "ours_p2p_nomc", {"RELORA_B200_MULTICAST": "0"})
        r3 = launch("ours", "ours_nccl", extra_args=("--comm", "nccl"))
        if bad(r3):
            launch("ours", "ours_nccl_nonvls", {"NCCL_NVLS_ENABLE": "0"}, extra_args=("--comm", "nccl"))
            launch("ours", "ours_nccl_nograph_native", extra_args=("--comm", "nccl", "--cuda_graphs", "false", "--attention", "native"))
    launch("nccl", "nccl_stress")
    rr = launch("ref", "ref_default", {"NCCL_DEBUG": "INFO", "NCCL_DEBUG_SUBSYS": "INIT"})
    if bad(rr):
        launch("ref", "ref_nonvls", {"NCCL_NVLS_ENABLE": "0"})
        launch("nccl", "nccl_stress_nonvls", {"NCCL_NVLS_ENABLE": "0"})
    print("[hunt] summary: " + json.dumps(summary), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["ours", "ref", "nccl", "drive"])
    ap.add_argument("--tag", default="run")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--iters", type=int, default=600)
    ap.add_argument("--gpus", type=int, default=4)
    ap.add_argument("--model", default="llama_250m")
    ap.add_argument("--comm", default="auto")
    ap.add_argument("--cuda_graphs", default="true")
    ap.add_argument("--attention", default="auto")
    ap.add_argument("--ga", type=int, default=None)
    ap.add_argument("--emulate_world", type=int, default=1)
    ap.add_argument("--pinpoint_step", type=int, default=-1)
    ap.add_argument("--sdpa_backend", default="default", choices=["default", "cudnn", "flash", "efficient", "math"])
    a = ap.parse_args()
    {"ours": run_ours, "ref": run_ref, "nccl": run_nccl, "drive": drive}[a.mode](a)
