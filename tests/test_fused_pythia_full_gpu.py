"""Full-rank training on the fused Pythia (GPT-NeoX) executor (H100: -m gpu): selection, gradients and updates against the module
path, determinism, every GEMM call against the reference, and a warm-up followed by ReLoRA through the command line."""
import copy
import os
import sys

import pytest
import torch

from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
VOCAB = 1024


def _relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def _neox(hd=64, parallel=True, act="gelu", rotary_pct=0.25, hidden=None, seed=0, layers=2, **over):
    """A bare GPT-NeoX with random biases and LayerNorm affines (the module init leaves them at 0 / 1)."""
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig

    hidden = hidden or (512 if hd == 256 else 256)
    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=VOCAB, hidden_size=hidden, num_hidden_layers=layers,
                       num_attention_heads=hidden // hd, intermediate_size=4 * hidden, rotary_pct=rotary_pct,
                       max_position_embeddings=128, layer_norm_eps=1e-5, use_parallel_residual=parallel, hidden_act=act,
                       rotary_emb_base=10000, tie_word_embeddings=False, **over)
    torch.manual_seed(seed)
    m = GPTNeoXForCausalLM(cfg)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias"):
                p.normal_(std=0.02)
            elif "layernorm" in n or "layer_norm" in n:
                p.add_(torch.randn_like(p) * 0.05)
    return m.cuda().to(BF).train()


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _fused(model, **kw):
    from relora_b200.engine.fused_pythia import FusedPythiaStepper

    kw.setdefault("lr", 1e-3)
    kw.setdefault("grad_accumulation", 1)
    return FusedPythiaStepper(model, _info(), **kw)


def _module(model, **kw):
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    kw.setdefault("lr", 1e-3)
    kw.setdefault("grad_accumulation", 1)
    return ModuleStepper(model, _info(), native=fused.NativeOptim() if next(model.parameters()).dtype == BF else None, **kw)


def _grads(st):
    return {n: st.store.view_like(st.store.grads, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


def _args(engine, **over):
    from argparse import Namespace

    kw = dict(engine=engine, optimizer="adam", comm="auto", lr=1e-3, adam_beta1=0.9, adam_beta2=0.999, weight_decay=0.0,
              clip_grad_norm=1.0, gradient_accumulation=1, cuda_graphs=False, attention="auto", frozen_dtype=None,
              deterministic=False)
    kw.update(over)
    return Namespace(**kw)


def test_selection():
    """`auto` keeps full-rank Pythia on the module path; `fused` builds the full-rank executor or names why it cannot."""
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.engine.stepper import ModuleStepper, make_stepper

    assert type(make_stepper(_neox(), _info(), _args("auto"))) is ModuleStepper
    st = make_stepper(_neox(), _info(), _args("fused", deterministic=True))
    assert type(st) is FusedPythiaStepper and st.full and st.wgrad_split_k == 1
    with pytest.raises(RuntimeError, match="not applicable: only the GELU activation is fused"):
        make_stepper(_neox(act="relu"), _info(), _args("fused"))
    with pytest.raises(RuntimeError, match="no frozen weights"):
        make_stepper(_neox(), _info(), _args("fused", frozen_dtype="fp8"))


def test_views_alias_the_module_parameters_and_merge_is_refused():
    m = _neox()
    st = _fused(m, cuda_graphs=False)
    h, f = 256, 1024
    for layer, S in zip(m.gpt_neox.layers, st.layers):
        at, mlp = layer.attention, layer.mlp
        for W, gW, b, mod, shape in ((S.W_qkv, S.gW_qkv, S.b_qkv, at.query_key_value, (3 * h, h)), (S.W_o, S.gW_o, S.b_o, at.dense, (h, h)),
                                     (S.W_h, S.gW_h, S.b_h, mlp.dense_h_to_4h, (f, h)), (S.W_4, S.gW_4, S.b_4, mlp.dense_4h_to_h, (h, f))):
            assert W.shape == shape and gW.shape == shape and gW.dtype == torch.float32
            assert W.data_ptr() == mod.weight.data_ptr() and mod.weight.is_contiguous() and b.data_ptr() == mod.bias.data_ptr()
            assert mod.weight.requires_grad
        assert S.A_qkv is None and S.gA_4 is None
    assert st.lora_params == [] and st.r == 0 and st.p == 0.0
    assert st.wgrad_split_k == 0  # split-K weight gradients unless --deterministic
    st.micro_step(torch.randint(0, VOCAB, (2, 64), device="cuda"))
    assert all(u is None for u in st.u_qkv) and st.tmp_h is None and st.tmp_f is None and not hasattr(st, "du_bufs")
    with pytest.raises(RuntimeError, match="ReLoRA"):
        st.merge_and_reinit()


@pytest.mark.parametrize("parallel,act,graphs,attention,hd,rotary_pct", [
    (True, "gelu", False, "native", 64, 0.25),
    (True, "gelu", True, "sdpa", 64, 0.25),
    (False, "gelu_new", True, "native", 64, 0.25),
    (False, "gelu", False, "sdpa", 128, 0.5),
    (True, "gelu_new", True, "native", 128, 0.25),
    (True, "gelu", False, "sdpa", 256, 0.25),
    (False, "gelu", True, "native", 256, 0.5),
])
def test_gradients_match_the_fp32_module_path(parallel, act, graphs, attention, hd, rotary_pct):
    """One micro-step on identical weights (T 96, ragged).  Reference: the same model in fp32 on the module path.  Each fused
    gradient (and the loss) may be off by at most twice the bf16 module path's own error, with a floor of 1e-2.  The rotary
    fractions leave rot < head_dim."""
    mb = _neox(hd=hd, parallel=parallel, act=act, rotary_pct=rotary_pct)
    mf, m32 = copy.deepcopy(mb), copy.deepcopy(mb).float()
    ids = torch.randint(0, VOCAB, (2, 96), device="cuda")
    l32 = m32(input_ids=ids, labels=ids).loss
    l32.backward()
    g32 = {n: p.grad for n, p in m32.named_parameters()}
    ms = _module(mb)
    lb = ms.micro_step(ids)
    st = _fused(mf, cuda_graphs=graphs, attention=attention)
    assert st.native_attn == (attention == "native") and st.rot < hd and st.parallel == parallel and st.tanh == (act == "gelu_new")
    lf = st.micro_step(ids)
    e_mod, e_fus = abs(float(lb) - float(l32)) / float(l32), abs(float(lf) - float(l32)) / float(l32)
    assert e_fus <= max(2 * e_mod, 1e-2), ("loss", e_fus, e_mod)
    gb, gf = _grads(ms), _grads(st)
    assert set(gf) == set(g32)
    worst = 0.0
    for n in g32:
        e_mod, e_fus = _relerr(gb[n], g32[n]), _relerr(gf[n], g32[n])
        worst = max(worst, e_fus)
        assert e_fus <= max(2 * e_mod, 1e-2), (n, e_fus, e_mod)
    print(f"[pythia full rank] parallel={parallel} {act} graphs={graphs} {attention} hd={hd} rot={st.rot}: "
          f"worst gradient relative error {worst:.3g}")


def test_updates_track_the_module_path_and_save_with_hf_keys(tmp_path):
    """5 updates with gradient accumulation 2 (weight decay on, graphs on, sequential residual).  Each parameter's distance from an
    fp32 module-path run may be at most twice the bf16 module path's distance, with a floor of 1e-2; the module parameters (views
    of the store) save and load under the HF GPT-NeoX keys."""
    from relora_b200.models import GPTNeoXForCausalLM

    mb = _neox(parallel=False)
    mf, m32 = copy.deepcopy(mb), copy.deepcopy(mb).float()
    kw = dict(lr=1e-3, weight_decay=0.1, grad_accumulation=2)
    steppers = {"fp32": _module(m32, **kw), "module": _module(mb, **kw), "fused": _fused(mf, cuda_graphs=True, **kw)}
    g = torch.Generator(device="cuda").manual_seed(5)
    batches = [torch.randint(0, VOCAB, (2, 96), device="cuda", generator=g) for _ in range(10)]
    losses = {k: [] for k in steppers}
    for i, ids in enumerate(batches):
        for k, st in steppers.items():
            losses[k].append(float(st.micro_step(ids)))
            if i % 2 == 1:
                st.update()
    p32 = dict(m32.named_parameters())
    worst = 0.0
    for (n, pm), pf in zip(mb.named_parameters(), mf.parameters()):
        d_mod, d_fus = _relerr(pm, p32[n]), _relerr(pf, p32[n])
        worst = max(worst, d_fus)
        assert d_fus <= max(2 * d_mod, 1e-2), (n, d_fus, d_mod)
    assert abs(losses["fused"][-1] - losses["fp32"][-1]) <= max(2 * abs(losses["module"][-1] - losses["fp32"][-1]), 1e-2 * losses["fp32"][-1])
    print(f"[pythia full rank] after 5 updates: worst parameter relative distance from fp32 {worst:.3g}; final loss fused "
          f"{losses['fused'][-1]:.4f} module {losses['module'][-1]:.4f} fp32 {losses['fp32'][-1]:.4f}")
    before = {k: v.detach().clone() for k, v in mf.named_parameters()}
    assert "gpt_neox.layers.0.attention.query_key_value.weight" in before and "embed_out.weight" in before
    mf.save_pretrained(str(tmp_path / "m"))
    back = GPTNeoXForCausalLM.from_pretrained(str(tmp_path / "m"))
    sd = back.state_dict()
    for k, v in before.items():
        assert torch.equal(sd[k].cpu().to(v.dtype), v.cpu()), k
    # the trained model evaluates the same through the module path
    ids = batches[0]
    back = back.cuda().to(BF).eval()
    with torch.no_grad():
        lm = float(back(input_ids=ids, labels=ids).loss)
    assert abs(float(steppers["fused"].eval_loss(ids)) - lm) < 2e-2


def test_deterministic_mode_is_bit_reproducible():
    """`deterministic=True` (no split-K in the weight gradients): two runs from the same seed give bit-identical gradients and,
    after an update without clipping, bit-identical parameters, for the projection weights, embed_in and embed_out.  The 1-D
    gradients (LayerNorm γ / β and the projection biases) are column sums whose block partials meet in fp32 atomics, and are
    excluded."""
    ids = torch.randint(0, VOCAB, (3, 128), device="cuda")
    runs = []
    for _ in range(2):
        m = _neox(seed=3)
        st = _fused(m, cuda_graphs=True, deterministic=True, clip_grad_norm=0.0)
        assert st.wgrad_split_k == 1 and st.native_attn
        st.micro_step(ids)
        torch.cuda.synchronize()
        g = {n: v.clone() for n, v in _grads(st).items()}
        st.update()
        torch.cuda.synchronize()
        runs.append((g, {n: p.detach().clone() for n, p in m.named_parameters()}))
    checked = 0
    for n, v in runs[0][0].items():
        if v.dim() == 1:
            continue
        assert torch.equal(v, runs[1][0][n]), n
        assert torch.equal(runs[0][1][n], runs[1][1][n]), n
        checked += 1
    assert checked == 2 * 4 + 2


def test_relora_path_ignores_deterministic():
    """The ReLoRA Pythia path keeps its split-K weight gradients whatever the flag says."""
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.relora import ReLoRaModel

    w = ReLoRaModel(_neox().cpu().float(), r=128, lora_alpha=32, lora_dropout=0.1,
                    target_modules=["attn", "attention", "mlp"]).cuda().to(BF)
    st = FusedPythiaStepper(w, _info(), lr=1e-3, cuda_graphs=False, deterministic=True)
    assert not st.full and st.wgrad_split_k == 0


# the GEMM modes of one full-rank micro-step and evaluation: projections with the bias (and residual) epilogue, input gradients
# reading W MN-major, fp32 weight gradients accumulated from two MN-major operands (split-K unless deterministic); no K2 (LoRA)
# segment, no per-group windows, no fp8
_FULL_MODES = {"bias", "residual", "b1_mn", "a1_mn", "accumulate", "split_k"}


@pytest.mark.parametrize("deterministic", [False, True])
def test_every_gemm_call_matches_the_reference(deterministic, monkeypatch):
    """Every gemm call of one full-rank micro-step and one evaluation (sequential residual, native attention), replayed on clones
    of its inputs against ops.reference.gemm_ref; the set of modes is the expected one, and no LoRA input-gradient kernel runs."""
    from relora_b200.ops import fused

    C = fused._C()
    st = _fused(_neox(parallel=False), cuda_graphs=False, deterministic=deterministic)
    gemm0 = fused.gemm
    seen = {"calls": 0, "worst": 0.0, "modes": set()}

    def audited(a1, b1, out=None, **kw):
        torch.cuda.synchronize()  # the weight gradients run on the side stream
        cl = lambda v: v.clone() if torch.is_tensor(v) else v  # noqa: E731
        a1c, b1c, kwc, prev = cl(a1), cl(b1), {k: cl(v) for k, v in kw.items()}, cl(out)
        res = gemm0(a1, b1, out, **kw)
        torch.cuda.synchronize()
        want, bound = ref.gemm_ref(a1c, b1c, prev, **kwc)
        seen["worst"] = max(seen["worst"], ref.assert_gemm_close(res, want, bound))
        seen["calls"] += 1
        for k, v in kw.items():
            if k == "split_k":
                if v != 1:
                    seen["modes"].add(k)
            elif k not in ("M", "N", "K1") and v is not None and v is not False and not (type(v) in (int, float) and v == 0):
                seen["modes"].add(k)
        return res

    def no_lora_dx(*a, **k):
        raise AssertionError("full-rank training has no LoRA input gradient")

    monkeypatch.setattr(fused, "gemm", audited)
    monkeypatch.setattr(C, "lora_dx", no_lora_dx)
    ids = torch.randint(0, VOCAB, (3, 97), device="cuda")
    loss = st.micro_step(ids)
    n_train = seen["calls"]
    ev = st.eval_loss(ids)
    assert torch.isfinite(loss) and torch.isfinite(ev)
    print(f"[gemm modes] pythia full rank deterministic={deterministic}: {seen['calls']} calls, worst ratio {seen['worst']:.3g}, "
          f"modes {sorted(seen['modes'])}")
    assert seen["modes"] == (_FULL_MODES - {"split_k"} if deterministic else _FULL_MODES)
    # per layer: 4 projections, 4 input gradients, 4 weight gradients; LM head: 3 per 4096-token chunk
    assert n_train == 2 * 12 + 3 and seen["calls"] - n_train == 2 * 4 + 1


def test_warmup_then_relora_through_the_command_line(tmp_path):
    """A tiny Pythia trains full-rank on the fused executor (--deterministic) and saves under the HF keys; ReLoRA continues from
    it as --warmed_up_model on the fused Pythia executor."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_neox_data import _tiny_pythia_dir
    from torchrun_main import main

    from relora_b200.models import GPTNeoXForCausalLM

    ckpt = _tiny_pythia_dir(str(tmp_path / "pythia-tiny"), hidden=128, heads=2)
    warm, rel = str(tmp_path / "warm"), str(tmp_path / "relora")
    common = ["--model_name_or_path", ckpt, "--synthetic_data", "512", "--batch_size", "4", "--total_batch_size", "8",
              "--max_length", "64", "--lr", "1e-3", "--warmup_steps", "2", "--eval_every", "100", "--dtype", "bfloat16",
              "--workers", "0", "--engine", "fused"]
    res = main(common + ["--scheduler", "cosine", "--num_training_steps", "8", "--save_every", "8", "--save_dir", warm,
                         "--deterministic", "true"])
    assert res["executor"] == "FusedPythiaStepper" and res["update_step"] == 8
    assert torch.isfinite(torch.tensor(res["final_eval_loss"]))
    saved = os.path.join(warm, "model_8")
    start, trained = GPTNeoXForCausalLM.from_pretrained(ckpt), GPTNeoXForCausalLM.from_pretrained(saved)
    w0 = start.state_dict()["gpt_neox.layers.0.attention.query_key_value.weight"]
    w1 = trained.state_dict()["gpt_neox.layers.0.attention.query_key_value.weight"]
    assert w1.shape == w0.shape and not torch.equal(w0.float(), w1.float())  # the projection weights trained

    res2 = main(common + ["--use_peft", "--lora_r", "128", "--relora", "4", "--cycle_length", "4", "--restart_warmup_steps", "1",
                          "--scheduler", "cosine_restarts", "--init_lora_a", "kaiming", "--warmed_up_model", saved,
                          "--num_training_steps", "16", "--save_every", "100", "--save_dir", rel])
    assert res2["executor"] == "FusedPythiaStepper" and res2["update_step"] == 16 and res2["n_lora_restarts"] >= 1
    assert torch.isfinite(torch.tensor(res2["final_eval_loss"]))
