"""Fused whole-model executor vs the module-by-module path on identical weights / dropout masks (H100: -m gpu)."""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


def _build(p_drop, seed=0, inter=512):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="llama", vocab_size=4096, hidden_size=256, intermediate_size=inter, num_hidden_layers=2,
                       num_attention_heads=4, rms_norm_eps=1e-6, pad_token_id=-1, max_position_embeddings=256)
    torch.manual_seed(seed)
    m = LlamaForCausalLM(cfg)
    w = ReLoRaModel(m, r=128, lora_alpha=32, lora_dropout=p_drop, target_modules=["attn", "mlp"], init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


@pytest.mark.parametrize("p_drop,graphs,inter", [(0.0, False, 512), (0.1, False, 512), (0.0, True, 512), (0.1, True, 512),
                                                  (0.1, True, 341), (0.0, False, 341)])
def test_fused_matches_module_path(p_drop, graphs, inter):
    """``inter=341`` exercises the zero-padded MLP blocks used for llama_1b (intermediate 5461 -> 5504)."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    wa = _build(p_drop, inter=inter)
    wb = copy.deepcopy(wa)
    ids = torch.randint(0, 4096, (3, 64), device=dev)
    fs = FusedLlamaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs)
    ms = ModuleStepper(wb, _info(), lr=1e-3, grad_accumulation=1, native=fused.NativeOptim())
    fused.seed_state.set(dev, 4321)
    la = fs.micro_step(ids)
    if graphs:  # a second replay accumulates a second gradient: compare after exactly one
        pass
    fused.seed_state.set(dev, 4321)
    lb = ms.micro_step(ids)
    assert abs(float(la) - float(lb)) < 4e-2, (float(la), float(lb))
    ga = {n: fs.store.view_like(fs.store.grads, p).float() for n, p in zip(fs.trainable_names, fs.trainable_params)}
    gb = {n: ms.store.view_like(ms.store.grads, p).float() for n, p in zip(ms.trainable_names, ms.trainable_params)}
    worst = 0.0
    for n in ga:
        if gb[n].norm() == 0:
            continue
        e = _relerr(ga[n], gb[n])
        worst = max(worst, e)
        assert e < 0.15, (n, e)
    # update + second micro-step runs (graph replay path) and changes the parameters
    before = fs.store.params.clone()
    fs.update()
    assert not torch.equal(before, fs.store.params)
    l2 = fs.micro_step(ids)
    assert torch.isfinite(l2)
    ev = fs.eval_loss(ids)
    assert torch.isfinite(ev) and abs(float(ev) - float(l2)) < 0.5


@pytest.mark.parametrize("inter", [512, 341])
def test_fused_merge_and_checkpoint_roundtrip(tmp_path, inter):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.relora import ReLoRaModel

    w = _build(0.1, inter=inter)
    fs = FusedLlamaStepper(w, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False)
    ids = torch.randint(0, 4096, (2, 64), device="cuda")
    w.eval()
    before = fs.eval_loss(ids)
    q = w.wrapped_model.model.layers[0].self_attn.q_proj
    want = (q.weight.float() + q.scaling * q.lora_B.weight.float() @ q.lora_A.weight.float())
    fs.merge_and_reinit()
    assert _relerr(q.weight, want) < 4e-3
    assert float(q.lora_B.weight.abs().sum()) == 0
    dn = w.wrapped_model.model.layers[1].mlp.down_proj
    assert dn.weight.shape == (256, inter) and float(dn.lora_A.weight.abs().sum()) > 0
    after = fs.eval_loss(ids)
    assert abs(float(before) - float(after)) < 3e-2
    # parameters are views of the stacked buffers, checkpoints still have the reference layout
    d = str(tmp_path / "m")
    w.save_pretrained(d)
    w2 = ReLoRaModel.from_pretrained(d)
    sd = w.wrapped_model.state_dict()
    for k, v in w2.wrapped_model.state_dict().items():
        assert torch.equal(v.cpu(), sd[k].cpu()), k


def test_native_attention_matches_sdpa_in_the_executor():
    """The wgmma attention kernels and torch SDPA (cuDNN) give the same loss and gradients inside the fused executor."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    wa = _build(0.1)
    wb = copy.deepcopy(wa)
    ids = torch.randint(0, 4096, (3, 128), device=dev)
    fa = FusedLlamaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=True, attention="native")
    fb = FusedLlamaStepper(wb, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False, attention="sdpa")
    assert fa.native_attn and not fb.native_attn
    fused.seed_state.set(dev, 77)
    la = fa.micro_step(ids)
    fused.seed_state.set(dev, 77)
    lb = fb.micro_step(ids)
    assert abs(float(la) - float(lb)) < 2e-2
    for n, p in zip(fa.trainable_names, fa.trainable_params):
        ga = fa.store.view_like(fa.store.grads, p).float()
        gb = fb.store.view_like(fb.store.grads, fb.trainable_params[fa.trainable_names.index(n)]).float()
        if gb.norm() == 0:
            continue
        assert _relerr(ga, gb) < 0.1, n


@pytest.mark.parametrize("backward", [False, True])
def test_fp8_frozen_path_tracks_bf16_executor(backward, monkeypatch):
    """--frozen_dtype fp8: E4M3 forward GEMMs for the frozen weights (delayed activation scaling) stay close to the bf16
    executor in loss and LoRA gradients, and keep working across an update and a merge."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    wa = _build(0.1)
    wb = copy.deepcopy(wa)
    ids = torch.randint(0, 4096, (3, 128), device=dev)
    if backward:  # E5M2 output gradients x E4M3 Wᵀ for the input-gradient GEMMs; lower the two-kernel threshold so the tiny model uses it
        monkeypatch.setenv("RELORA_B200_DX_SPLIT_K", "512")
    fa = FusedLlamaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=True, fp8=True, fp8_backward=backward)
    fb = FusedLlamaStepper(wb, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False)
    assert fa.fp8 and not fb.fp8 and fa.fp8_bwd == backward
    fused.seed_state.set(dev, 5)
    la = fa.micro_step(ids)   # the capture warm-up has already calibrated the activation scales
    fused.seed_state.set(dev, 5)
    lb = fb.micro_step(ids)
    assert abs(float(la) - float(lb)) < 5e-2, (float(la), float(lb))
    worst = 0.0
    for n, p in zip(fa.trainable_names, fa.trainable_params):
        if "lora_" not in n:
            continue
        ga = fa.store.view_like(fa.store.grads, p).float()
        gb = fb.store.view_like(fb.store.grads, fb.trainable_params[fa.trainable_names.index(n)]).float()
        if gb.norm() == 0:
            continue
        worst = max(worst, _relerr(ga, gb))
    assert worst < (0.4 if backward else 0.25), worst
    fa.update()
    fa.merge_and_reinit()
    l2 = fa.micro_step(ids)
    assert torch.isfinite(l2) and abs(float(l2) - float(la)) < 1.0


@pytest.mark.parametrize("extra", [[], ["--frozen_dtype", "fp8", "--attention", "native"]])
def test_cli_end_to_end_on_the_fused_executor(tmp_path, extra):
    """torchrun_main on the H100 executor: ReLoRA resets, magnitude pruning, checkpoint layout, autoresume; also with the fp8
    frozen-weight path and the wgmma attention kernels selected from the command line."""
    import json
    import os

    from torchrun_main import main

    cfg = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "vocab_size": 4096, "hidden_size": 256, "intermediate_size": 512,
           "num_hidden_layers": 2, "num_attention_heads": 4, "rms_norm_eps": 1e-6, "max_sequence_length": 256, "hidden_act": "silu",
           "bos_token_id": 0, "eos_token_id": 1, "pad_token_id": -1, "initializer_range": 0.02, "use_cache": True}
    cfg_path = str(tmp_path / "llama_tiny.json")
    json.dump(cfg, open(cfg_path, "w"))
    d = str(tmp_path / "run")
    args = ["--model_config", cfg_path, "--synthetic_data", "4096", "--batch_size", "4", "--total_batch_size", "8", "--max_length", "128",
            "--lr", "1e-3", "--use_peft", "--lora_r", "128", "--relora", "4", "--cycle_length", "4", "--restart_warmup_steps", "1",
            "--scheduler", "cosine_restarts", "--warmup_steps", "2", "--num_training_steps", "8", "--save_every", "4",
            "--eval_every", "100", "--save_dir", d, "--dtype", "bfloat16", "--workers", "0", "--optimizer_magnitude_pruning", "0.9",
            "--reset_optimizer_on_relora", "false",
            "--init_lora_a", "kaiming", *extra]
    res = main(args)
    assert res["executor"] == "FusedLlamaStepper" and res["update_step"] == 8
    assert res["n_lora_restarts"] == 1 and res["n_optimizer_resets"] == 1
    assert torch.isfinite(torch.tensor(res["final_eval_loss"])) and res["final_eval_loss"] < 9.0
    for f in ("config.json", "pytorch_model.bin", "relora_config.json", "optimizer.pt", "training_state.json"):
        assert os.path.exists(os.path.join(d, "model_8", f)), f
    # autoresume picks up the last checkpoint and continues to a longer horizon
    res2 = main(args + ["--autoresume", "true", "--num_training_steps", "12"])
    assert res2["update_step"] == 12 and "model_12" in os.listdir(d)


@pytest.mark.parametrize("quant", ["8bit", "4bit"])
def test_cli_quantized_frozen_weights_train_on_packed_storage(tmp_path, quant):
    """`--quantize 8bit|4bit` (reference: bitsandbytes int8 / NF4, relora.py:222-238): the frozen weights are resident only as packed
    bytes + block scales; 8bit runs the block-scaled MXFP8 tensor-core GEMMs (csrc/gemm_mx.cu), a merge requantises in place, and the
    checkpoint keeps the reference layout (dense `weight` entries)."""
    import json
    import os

    from torchrun_main import main

    cfg = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "vocab_size": 4096, "hidden_size": 256, "intermediate_size": 512,
           "num_hidden_layers": 2, "num_attention_heads": 4, "rms_norm_eps": 1e-6, "max_sequence_length": 256, "hidden_act": "silu",
           "bos_token_id": 0, "eos_token_id": 1, "pad_token_id": -1, "initializer_range": 0.02, "use_cache": True}
    cfg_path = str(tmp_path / "llama_tiny.json")
    json.dump(cfg, open(cfg_path, "w"))
    d = str(tmp_path / "run")
    args = ["--model_config", cfg_path, "--synthetic_data", "4096", "--batch_size", "4", "--total_batch_size", "8", "--max_length", "128",
            "--lr", "1e-3", "--use_peft", "--lora_r", "128", "--relora", "4", "--cycle_length", "4", "--restart_warmup_steps", "1",
            "--scheduler", "cosine_restarts", "--warmup_steps", "2", "--num_training_steps", "8", "--save_every", "8",
            "--eval_every", "100", "--save_dir", d, "--dtype", "bfloat16", "--workers", "0", "--init_lora_a", "kaiming", "--quantize", quant]
    res = main(args)
    assert res["executor"] == "ModuleStepper" and res["update_step"] == 8 and res["n_lora_restarts"] == 1
    assert torch.isfinite(torch.tensor(res["final_eval_loss"])) and res["final_eval_loss"] < 9.0
    sd = torch.load(os.path.join(d, "model_8", "pytorch_model.bin"), weights_only=True)
    w = sd["model.layers.0.self_attn.q_proj.weight"]
    assert w.shape == (256, 256) and bool(torch.isfinite(w.float()).all())


def test_deterministic_mode_reproduces_lora_and_embedding_gradients_bit_for_bit():
    """`--deterministic`: weight-gradient GEMMs without split-K atomics + the sorted embedding backward -> two runs of the same
    micro-batch give bit-identical LoRA / embedding / LM-head gradients (the default split-K path may differ in the last bits)."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    ids = torch.randint(0, 4095, (3, 128), device=dev)
    grads = []
    for _ in range(2):
        w = _build(0.1, seed=3)
        fs = FusedLlamaStepper(w, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False, deterministic=True)
        fused.seed_state.set(dev, 99)
        fs.micro_step(ids)
        torch.cuda.synchronize()
        grads.append({n: fs.store.view_like(fs.store.grads, p).clone() for n, p in zip(fs.trainable_names, fs.trainable_params)})
    for n in grads[0]:
        if "layernorm" in n or n.endswith("norm.weight"):
            continue  # [h]-sized norm gradients are combined with vector atomics (documented)
        assert torch.equal(grads[0][n], grads[1][n]), n
