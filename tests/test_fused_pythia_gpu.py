"""Pythia (GPT-NeoX) fused executor vs the module path on identical weights and dropout masks, and its kernels (H100: -m gpu)."""
import copy
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


def _build(p_drop=0.1, hd=64, parallel=True, act="gelu", max_pos=64, seed=0, hidden=256):
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=1024, hidden_size=hidden, num_hidden_layers=2, num_attention_heads=hidden // hd,
                       intermediate_size=4 * hidden, rotary_pct=0.25, max_position_embeddings=max_pos, layer_norm_eps=1e-5,
                       use_parallel_residual=parallel, hidden_act=act, rotary_emb_base=10000, tie_word_embeddings=False)
    torch.manual_seed(seed)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=p_drop, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming")
    with torch.no_grad():
        for mod in w.relora_modules():
            torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
            torch.nn.init.normal_(mod.bias, std=0.02)
        for n, p in w.named_parameters():
            if "layernorm" in n or "layer_norm" in n:
                p.add_(torch.randn_like(p) * 0.05)
    return w.cuda().to(BF).train()


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _grads(st):
    return {n: st.store.view_like(st.store.grads, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


@pytest.mark.parametrize("p_drop,graphs,parallel,hd,T,act", [
    (0.0, False, True, 64, 96, "gelu"),
    (0.1, False, True, 64, 96, "gelu"),
    (0.1, True, True, 64, 96, "gelu"),
    (0.0, True, True, 128, 80, "gelu_new"),
    (0.1, False, False, 64, 96, "gelu"),
    (0.1, True, False, 128, 80, "gelu"),
    (0.1, True, True, 128, 50, "gelu_new"),
    (0.0, False, False, 64, 50, "gelu_new"),
])
def test_fused_pythia_matches_module_path(p_drop, graphs, parallel, hd, T, act):
    """T = 96 / 80 are ragged and beyond max_position_embeddings (64); gelu_new is the tanh form."""
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    wa = _build(p_drop, hd=hd, parallel=parallel, act=act)
    wb = copy.deepcopy(wa)
    ids = torch.randint(0, 1024, (2, T), device=dev)
    fs = FusedPythiaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs)
    ms = ModuleStepper(wb, _info(), lr=1e-3, grad_accumulation=1, native=fused.NativeOptim())
    fused.seed_state.set(dev, 4321)
    la = fs.micro_step(ids)
    fused.seed_state.set(dev, 4321)
    lb = ms.micro_step(ids)
    assert abs(float(la) - float(lb)) < 4e-2, (float(la), float(lb))
    ga, gb = _grads(fs), _grads(ms)
    assert set(ga) == set(gb)
    for n in ga:
        if gb[n].norm() == 0:
            continue
        assert _relerr(ga[n], gb[n]) < 0.15, (n, _relerr(ga[n], gb[n]))
    for key in ("query_key_value.bias", "dense_4h_to_h.bias", "input_layernorm.bias", "embed_in.weight", "embed_out.weight"):
        assert any(key in n and gb[n].norm() > 0 for n in gb), key
    before = fs.store.params.clone()
    fs.update()
    assert not torch.equal(before, fs.store.params)
    l2 = fs.micro_step(ids)  # graph replay when graphs are on
    assert torch.isfinite(l2)
    wb.load_state_dict(wa.state_dict())
    wb.eval()  # no LoRA dropout in the module path's evaluation either
    assert abs(float(fs.eval_loss(ids)) - float(ms.eval_loss(ids))) < 4e-2


@pytest.mark.parametrize("hd", [64, 128, 256])
def test_native_attention_matches_sdpa_in_the_pythia_executor(hd):
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    wa = _build(0.1, hd=hd, hidden=512 if hd == 256 else 256)
    wb = copy.deepcopy(wa)
    ids = torch.randint(0, 1024, (2, 160), device=dev)
    fa = FusedPythiaStepper(wa, _info(), lr=1e-3, cuda_graphs=True, attention="native")
    fb = FusedPythiaStepper(wb, _info(), lr=1e-3, cuda_graphs=False, attention="sdpa")
    assert fa.native_attn and not fb.native_attn
    fused.seed_state.set(dev, 77)
    la = fa.micro_step(ids)
    fused.seed_state.set(dev, 77)
    lb = fb.micro_step(ids)
    assert abs(float(la) - float(lb)) < 2e-2
    ga, gb = _grads(fa), _grads(fb)
    for n in ga:
        if gb[n].norm() > 0:
            assert _relerr(ga[n], gb[n]) < 0.1, n


@pytest.mark.parametrize("hd", [64, 128, 256])
def test_interleaved_layout_is_a_permutation_of_the_default(hd):
    """Same q, k, v in the two head layouts: bit-identical outputs, lse and (permuted) gradients."""
    import relora_b200._C as C

    B, T, nh = 2, 150, 3
    torch.manual_seed(hd)
    q, k, v = (torch.randn(B, T, nh, hd, device="cuda", dtype=BF) for _ in range(3))
    do = torch.randn(B * T, nh * hd, device="cuda", dtype=BF)
    std = torch.stack([q, k, v], 2).reshape(B * T, 3 * nh * hd).contiguous()     # [(q|k|v), nh, hd]
    il = torch.stack([q, k, v], 3).reshape(B * T, 3 * nh * hd).contiguous()      # [nh, (q|k|v), hd]
    res = {}
    for name, buf, flag in (("std", std, False), ("il", il, True)):
        out = torch.full((B * T, nh * hd), float("nan"), device="cuda", dtype=BF)
        lse = torch.empty(B, nh, T, device="cuda")
        C.attention_fwd(buf, out, lse, B, T, nh, hd, hd ** -0.5, interleaved=flag)
        d = torch.full_like(buf, float("nan"))
        C.attention_bwd(buf, out, do, lse, torch.empty_like(lse), d, B, T, nh, hd, hd ** -0.5, interleaved=flag)
        res[name] = (out, lse, d)
    assert torch.equal(res["std"][0], res["il"][0]) and torch.equal(res["std"][1], res["il"][1])
    d_std = res["std"][2].view(B * T, 3, nh, hd)
    d_il = res["il"][2].view(B * T, nh, 3, hd).transpose(1, 2)
    assert torch.equal(d_std, d_il)


@pytest.mark.parametrize("H,M", [(256, 77), (768, 130), (2048, 33)])
@pytest.mark.parametrize("parallel", [True, False])
def test_layernorm_executor_kernels_vs_fp32(H, M, parallel):
    import relora_b200._C as C
    from relora_b200.ops import reference as ref

    torch.manual_seed(H + M)
    dev = "cuda"
    x = (torch.randn(M, H, device=dev) * 2 + 0.5).to(BF)
    w1, b1, w2, b2 = ((torch.randn(H, device=dev) * 0.2 + (1.0 if i % 2 == 0 else 0.0)).to(BF) for i in range(4))
    p, seed_val, keys = 0.1, 1234, [7, 9]
    seed = torch.tensor([seed_val], dtype=torch.int32, device=dev)
    y1, y2, xd1, xd2 = (torch.empty(M, H, device=dev, dtype=BF) for _ in range(4))
    mean, rstd = torch.empty(M, device=dev), torch.empty(M, device=dev)
    kw = dict(w2=w2, b2=b2, y2=y2, xd2=xd2) if parallel else {}
    C.layernorm_fwd(x, w1, b1, y1, mean, rstd, 1e-5, xd=xd1, seed=seed, keys=keys, p=p, **kw)
    xf = x.float()
    ln = lambda w, b: torch.nn.functional.layer_norm(xf, (H,), w.float(), b.float(), 1e-5)  # noqa: E731
    assert _relerr(y1, ln(w1, b1)) < 1e-2
    m1 = ref.dropout_keep_mask(ref.mix_seed(seed_val, keys[0]), M, H, p, device=dev)
    assert torch.equal(xd1, (y1.float() * m1 / (1 - p)).to(BF))
    if parallel:
        assert _relerr(y2, ln(w2, b2)) < 1e-2
        m2 = ref.dropout_keep_mask(ref.mix_seed(seed_val, keys[1]), M, H, p, device=dev)
        assert torch.equal(xd2, (y2.float() * m2 / (1 - p)).to(BF))
    # backward: dx = dres + LN1ᵀ(dy1) [+ LN2ᵀ(dy2)], γ / β gradients, Σ rows of dres
    dy1, dy2, dres = (torch.randn(M, H, device=dev).to(BF) for _ in range(3))
    xr = xf.clone().requires_grad_()
    p1 = [w1.float().requires_grad_(), b1.float().requires_grad_()]
    p2 = [w2.float().requires_grad_(), b2.float().requires_grad_()]
    loss = (torch.nn.functional.layer_norm(xr, (H,), *p1, 1e-5) * dy1.float()).sum()
    if parallel:
        loss = loss + (torch.nn.functional.layer_norm(xr, (H,), *p2, 1e-5) * dy2.float()).sum()
    loss.backward()
    dx_want = xr.grad + dres.float()
    g = [torch.zeros(H, device=dev) for _ in range(6)]
    dx = torch.empty(M, H, device=dev, dtype=BF)
    kw = dict(dy2=dy2, w2=w2, dw2=g[2], db2=g[3], dres_sum2=g[5]) if parallel else {}
    C.layernorm_bwd(dy1, x, w1, mean, rstd, dx, g[0], g[1], dres=dres, dres_sum=g[4], **kw)
    assert _relerr(dx, dx_want) < 1e-2
    assert _relerr(g[0], p1[0].grad) < 1e-3 and _relerr(g[1], p1[1].grad) < 1e-3
    assert _relerr(g[4], dres.float().sum(0)) < 1e-4
    if parallel:
        assert _relerr(g[2], p2[0].grad) < 1e-3 and _relerr(g[3], p2[1].grad) < 1e-3
        assert torch.equal(g[4], g[5])


@pytest.mark.parametrize("tanh", [False, True])
def test_gelu_dropout_copy_and_bias_gradient(tanh):
    import relora_b200._C as C
    from relora_b200.ops import reference as ref

    M, N = 97, 1024
    z = torch.randn(M, N, device="cuda").to(BF)
    a, xd, dz = (torch.empty_like(z) for _ in range(3))
    seed = torch.tensor([99], dtype=torch.int32, device="cuda")
    C.gelu_fwd(z, a, tanh, xd=xd, seed=seed, key=5, p=0.1)
    want = torch.nn.functional.gelu(z.float(), approximate="tanh" if tanh else "none")
    assert _relerr(a, want) < 1e-2
    keep = ref.dropout_keep_mask(ref.mix_seed(99, 5), M, N, 0.1, device="cuda")
    assert torch.equal(xd, (a.float() * keep / 0.9).to(BF))
    da = torch.randn(M, N, device="cuda").to(BF)
    dz0 = torch.empty_like(z)
    C.gelu_bwd(da, z, dz0, tanh)
    db = torch.zeros(N, device="cuda")
    C.gelu_bwd(da, z, dz, tanh, dbias=db)
    assert torch.equal(dz, dz0)
    assert _relerr(db, dz.float().sum(0)) < 1e-4
    cs = torch.zeros(N, device="cuda")
    C.colsum(da, cs)
    C.colsum(da, cs)
    assert _relerr(cs, 2 * da.float().sum(0)) < 1e-4


def test_pythia_merge_and_checkpoint_roundtrip(tmp_path):
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.relora import ReLoRaModel

    w = _build(0.1)
    fs = FusedPythiaStepper(w, _info(), lr=1e-3, cuda_graphs=False)
    ids = torch.randint(0, 1024, (2, 64), device="cuda")
    before = fs.eval_loss(ids)
    q = w.wrapped_model.gpt_neox.layers[0].attention.query_key_value
    want = q.weight.float() + q.scaling * q.lora_B.weight.float() @ q.lora_A.weight.float()
    fs.merge_and_reinit()
    assert _relerr(q.weight, want) < 4e-3
    assert float(q.lora_B.weight.abs().sum()) == 0 and float(q.lora_A.weight.abs().sum()) > 0
    assert abs(float(before) - float(fs.eval_loss(ids))) < 3e-2
    d = str(tmp_path / "m")
    w.save_pretrained(d)
    w2 = ReLoRaModel.from_pretrained(d)
    sd = w.wrapped_model.state_dict()
    sd2 = w2.wrapped_model.state_dict()
    assert set(sd2) == set(sd) and "gpt_neox.layers.0.attention.query_key_value.lora_A.weight" in sd
    for k, v in sd2.items():
        assert torch.equal(v.cpu(), sd[k].cpu()), k


def test_auto_keeps_pythia_on_the_module_path_and_fused_selects_the_executor():
    from argparse import Namespace

    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.engine.stepper import ModuleStepper, make_stepper

    args = dict(optimizer="adam", lr=1e-3, adam_beta1=0.9, adam_beta2=0.999, weight_decay=0.0, clip_grad_norm=1.0,
                gradient_accumulation=1, comm="auto", cuda_graphs=False, attention="auto")
    assert type(make_stepper(_build(), _info(), Namespace(engine="auto", **args))) is ModuleStepper
    assert type(make_stepper(_build(), _info(), Namespace(engine="fused", **args))) is FusedPythiaStepper
    with pytest.raises(RuntimeError, match="GELU"):
        make_stepper(_build(act="relu"), _info(), Namespace(engine="fused", **args))


def test_cli_pythia_recipe_on_the_fused_executor(tmp_path):
    """The toy form of the shipped recipe (Pythia warm start, Megatron data, magnitude pruning, autoresume) with --engine fused."""
    import yaml

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_neox_data import _tiny_pythia_dir, _write_corpus
    from torchrun_main import main

    ckpt = _tiny_pythia_dir(str(tmp_path / "pythia-tiny"), hidden=128, heads=2)
    prefix = str(tmp_path / "pile")
    _write_corpus(prefix, n_docs=400, vocab=512, seed=11)
    data = tmp_path / "data.yaml"
    data.write_text(yaml.safe_dump({"data-path": prefix, "split": "8,1,1", "data-impl": "mmap", "seq-length": 64, "train-iters": 20,
                                    "eval-interval": 5, "eval-iters": 1}))
    recipe = tmp_path / "recipe.yaml"
    recipe.write_text(yaml.safe_dump(dict(
        model_name_or_path=ckpt, model_revision="step1000", dtype="bfloat16", distributed_type="ddp",
        megatron_dataset_config=str(data), max_length=64, workers=0,
        use_peft=True, lora_r=128, relora=3, force_keep_original=True, restart_warmup_steps=1, reset_optimizer_on_relora=False,
        optimizer_magnitude_pruning=0.8, optimizer="adam", lr=4e-4, adam_beta1=0.9, adam_beta2=0.95, weight_decay=0.01,
        scheduler="cosine_restarts", warmup_steps=2, batch_size=2, total_batch_size=4, num_training_steps=9,
        save_dir=str(tmp_path / "run"), autoresume=True, save_every=3, eval_every=3, tags="relora1b", comment="toy")))
    res = main(["--training_config", str(recipe), "--device", "cuda", "--engine", "fused"])
    assert res["executor"] == "FusedPythiaStepper" and res["update_step"] == 9 and res["n_lora_restarts"] == 2
    assert res["final_eval_loss"] < 7.5  # ln(512) = 6.24 at init
    recipe.write_text(recipe.read_text().replace("num_training_steps: 9", "num_training_steps: 12"))
    res2 = main(["--training_config", str(recipe), "--device", "cuda", "--engine", "fused"])
    assert res2["executor"] == "FusedPythiaStepper" and res2["update_step"] == 12
