"""Per-call-site roofline of the fused training step.

    python bench/site_profile.py [--model llama_250m] [--batch 24] [--seq 512] [--out gpurun_out/site_profile.json]

Every launch of this repo's extension inside one micro-step (+ the optimizer update) is tagged with its call site
(GEMM shape / operand majors / grouping, or the elementwise kernel's name), timed by the CUDA profiler (kineto kernel
durations, no graph, launches matched to tags by order) and compared against its roofline:

    t_min = max(flops / bf16_peak, bytes / hbm_bw)      (MEASURED_PEAKS.json; fallbacks: H100 SXM data sheet,
                                                           989 TFLOP/s dense BF16, 3.35 TB/s HBM3)

``bytes`` is the compulsory traffic (each operand once); ``frac`` = t_min / t_measured.  Library kernels (cuDNN
attention) are listed with their measured time only.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("RELORA_B200_NO_WANDB", "1")

from relora_b200.engine.api import TrainingEngine  # noqa: E402
from relora_b200.ops import fused  # noqa: E402
from relora_b200.parallel.dist import DistInfo  # noqa: E402


def peaks():
    try:
        d = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return float(d.get("bf16_tflops", 989.0)) * 1e12, float(d.get("hbm_gbs", 3350.0)) * 1e9
    except Exception:
        return 989e12, 3350e9


def tensor_bytes(args, kwargs):
    n = 0
    for v in list(args) + list(kwargs.values()):
        if isinstance(v, torch.Tensor):
            n += v.numel() * v.element_size()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="llama_250m")
    ap.add_argument("--batch", type=int, default=24)
    ap.add_argument("--seq", type=int, default=512)
    ap.add_argument("--out", default=None)
    ap.add_argument("--frozen_dtype", default=None)
    a = ap.parse_args()
    info = DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")
    torch.cuda.set_device(0)
    eng = TrainingEngine.build(
        info, model_config=os.path.join(ROOT, "configs", f"{a.model}.json"), batch_size=a.batch, gradient_accumulation=1,
        total_batch_size=a.batch, max_length=a.seq, use_peft=True, lora_r=128, relora=5000, cycle_length=5000,
        scheduler="cosine_restarts", warmup_steps=500, restart_warmup_steps=100, lr=1e-3, num_training_steps=20000,
        dtype="bfloat16", device="cuda", cuda_graphs=False, engine="fused", frozen_dtype=a.frozen_dtype)
    st = eng.stepper
    st.side = None  # serial launch order so kernels map to tags one to one
    C = st.C
    ids = torch.randint(0, 32000, (1, a.batch, a.seq), device="cuda")
    for _ in range(2):
        eng.train_step_device(ids)
    torch.cuda.synchronize()

    tags = []  # (tag, flops, bytes) per launch of the extension, in launch order

    real_gemm = fused.gemm

    def gemm_tagged(a1, b1, out, **kw):
        M = kw.get("M", a1.shape[0])
        N = kw.get("N", b1.shape[0])
        K1 = kw.get("K1", a1.shape[1])
        K2 = kw.get("K2", 0) if kw.get("a2") is not None else 0
        G = 1
        if kw.get("n_per_group"):
            G = N // kw["n_per_group"]
        if kw.get("m_per_group"):
            G = M // kw["m_per_group"]
        esz_out = out.element_size()
        e1 = 1.0 if kw.get("fp8") else 2.0  # bytes per element of segment 1
        flops = 2.0 * M * N * (K1 + K2)
        # compulsory bytes: A once, B once (grouped operands: every group's window once), output written (+read if accumulate)
        a_cols = K1 * (G if kw.get("a1_group_kofs") else 1)
        by = e1 * M * a_cols + e1 * N * K1 + 2.0 * (M * K2 * (G if kw.get("a2_group_kofs") else 1) + N * K2)
        by += esz_out * M * N * (2 if kw.get("accumulate") else 1)
        if kw.get("residual") is not None:
            by += 2.0 * M * N
        tag = "gemm M%d N%d K%d%s %s%s%s%s%s" % (
            M, N, K1, "+%d" % K2 if K2 else "", "A:mn " if kw.get("a1_mn") else "", "B:mn " if kw.get("b1_mn") else "",
            "G%d " % G if G > 1 else "", "acc32 " if kw.get("accumulate") and out.dtype == torch.float32 else "",
            ("+res" if kw.get("residual") is not None else "") + (" fp8" if kw.get("fp8") else ""))
        n0 = C.launch_count()
        r = real_gemm(a1, b1, out, **kw)
        for _ in range(C.launch_count() - n0):
            tags.append((tag.strip(), flops, by))
        return r

    class Tagger:
        def __init__(self, inner):
            self._inner = inner

        def __getattr__(self, name):
            fn = getattr(self._inner, name)
            if not callable(fn) or name in ("launch_count", "reset_launch_count"):
                return fn

            def wrapped(*args, **kw):
                n0 = self._inner.launch_count()
                r = fn(*args, **kw)
                dn = self._inner.launch_count() - n0
                if dn:
                    by = tensor_bytes(args, kw)
                    tag, fl = name, 0.0
                    if name in ("attention_fwd", "attention_bwd"):
                        Bq, Tq, nhq, hdq = (int(v) for v in (args[3:7] if name == "attention_fwd" else args[6:10]))
                        fwd = 2.0 * Bq * nhq * Tq * Tq * hdq  # causal: half of the 4·B·nh·T²·hd of S = QKᵀ and O = PV
                        fl = fwd if name == "attention_fwd" else 2.5 * fwd  # backward: 5 products instead of 2
                        tag = "%s B%d T%d nh%d hd%d" % (name, Bq, Tq, nhq, hdq)
                    if name == "lora_dx":
                        dy, w, du, aa, out = args[:5]
                        base = args[8] if len(args) > 8 else kw.get("base")
                        G = len(args[6])
                        Mx, N = out.shape
                        Kb = 0 if base is not None else dy.shape[1]
                        fl = 2.0 * Mx * N * (Kb + du.shape[1])
                        by = 2.0 * (Mx * Kb + Kb * N + Mx * du.shape[1] + du.shape[1] * N + Mx * N * (2 if base is not None else 1))
                        tag = "lora_dx M%d N%d Kb%d G%d%s" % (Mx, N, Kb, G, " (+base)" if base is not None else "")
                    for _ in range(dn):
                        tags.append((tag, fl / dn, by / dn))
                return r

            return wrapped

    fused.gemm = gemm_tagged
    st.C = Tagger(C)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        eng.train_step_device(ids)
        torch.cuda.synchronize()
    fused.gemm = real_gemm
    st.C = C

    kernels = []
    other = collections.defaultdict(lambda: [0.0, 0])
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        dur = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
        name = e.name
        if name.startswith("void rb::") or name.startswith("rb::"):
            kernels.append((e.time_range.start, name, dur))
        elif "Memcpy" in name or "Memset" in name or name.startswith("void") or "cudnn" in name or "kernel" in name:
            other[name[:90]][0] += dur
            other[name[:90]][1] += 1
    kernels.sort()
    # the optimizer (NativeOptim) launches through the un-tagged module handle; drop tags/kernels that do not pair up
    n = min(len(kernels), len(tags))
    peak_f, peak_b = peaks()
    agg = collections.OrderedDict()
    for (_, kname, dur), (tag, fl, by) in zip(kernels[:n], tags[:n]):
        key = tag
        d = agg.setdefault(key, {"site": key, "kernel": kname.split("(")[0][:60], "calls": 0, "us": 0.0, "flops": 0.0, "bytes": 0.0})
        d["calls"] += 1
        d["us"] += dur
        d["flops"] += fl
        d["bytes"] += by
    rows = []
    for d in agg.values():
        t = d["us"] * 1e-6
        tmin = max(d["flops"] / peak_f, d["bytes"] / peak_b)
        d["bound"] = "compute" if d["flops"] / peak_f >= d["bytes"] / peak_b else "memory"
        d["roofline_us"] = tmin * 1e6
        d["frac_of_roofline"] = tmin / t if t > 0 else None
        d["tflops"] = d["flops"] / t / 1e12 if t > 0 else 0.0
        d["gbps"] = d["bytes"] / t / 1e9 if t > 0 else 0.0
        rows.append(d)
    rows.sort(key=lambda d: -d["us"])
    tot = sum(d["us"] for d in rows)
    tot_min = sum(d["roofline_us"] for d in rows)
    lib = sorted(([k, v[0], v[1]] for k, v in other.items()), key=lambda r: -r[1])
    print(f"matched {n} launches (kernels {len(kernels)}, tags {len(tags)}); ours {tot/1e3:.2f} ms, roofline {tot_min/1e3:.2f} ms "
          f"({100*tot_min/tot:.1f}%), library/other {sum(r[1] for r in lib)/1e3:.2f} ms")
    print(f"{'site':58s} {'calls':>5s} {'ms':>8s} {'TFLOP/s':>8s} {'GB/s':>7s} {'bound':>7s} {'frac':>6s}")
    for d in rows:
        print(f"{d['site'][:58]:58s} {d['calls']:5d} {d['us']/1e3:8.3f} {d['tflops']:8.1f} {d['gbps']:7.0f} {d['bound']:>7s} "
              f"{(d['frac_of_roofline'] or 0):6.2f}")
    for k, t, c in lib[:12]:
        print(f"  other: {t/1e3:8.3f} ms x{c:<4d} {k}")
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        json.dump({"model": a.model, "batch": a.batch, "seq": a.seq, "peak_bf16_flops": peak_f, "peak_hbm_Bps": peak_b,
                   "ours_ms": tot / 1e3, "roofline_ms": tot_min / 1e3, "sites": rows, "other": lib[:20]}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
