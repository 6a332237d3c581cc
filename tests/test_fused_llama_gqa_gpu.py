"""The fused Llama executor with grouped-query attention (H100: -m gpu): against the module path on identical weights and dropout
masks, native vs SDPA attention inside it, every GEMM / lora_dx call audited against the reference, merge + checkpoint round trip,
and the CLI end to end from a Hugging Face format GQA checkpoint."""
import copy
import json
import os

import pytest
import torch

from test_gemm_modes_gpu import _GROUPED, _Audit

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


def _build(p_drop, inter=512, hidden=256, nh=4, nkv=2, seed=0):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="llama", vocab_size=4096, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=2,
                       num_attention_heads=nh, num_key_value_heads=nkv, rope_theta=500000.0, rms_norm_eps=1e-6, pad_token_id=-1,
                       max_position_embeddings=256)
    torch.manual_seed(seed)
    w = ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=p_drop, target_modules=["attn", "mlp"],
                    init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _grads(st):
    return {n: st.store.view_like(st.store.grads, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


# hidden 256 / 4 heads / 2 KV heads: head_dim 64, group 2; hidden 512 / 8 / 2: group 4; hidden 256 / 2 / 1: head_dim 128
@pytest.mark.parametrize("p_drop,graphs,inter,shape", [(0.0, False, 512, (256, 4, 2)), (0.1, False, 512, (256, 4, 2)),
                                                        (0.0, True, 512, (256, 4, 2)), (0.1, True, 512, (512, 8, 2)),
                                                        (0.1, True, 341, (256, 4, 2)), (0.0, False, 341, (256, 2, 1))])
def test_fused_gqa_matches_module_path(p_drop, graphs, inter, shape):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    hidden, nh, nkv = shape
    dev = torch.device("cuda", 0)
    wa = _build(p_drop, inter, hidden, nh, nkv)
    wb = copy.deepcopy(wa)
    ids = torch.randint(0, 4096, (3, 64), device=dev)
    fs = FusedLlamaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs, attention="native")
    ms = ModuleStepper(wb, _info(), lr=1e-3, grad_accumulation=1, native=fused.NativeOptim())
    assert fs.Wqkv.shape == (2, hidden + 2 * nkv * hidden // nh, hidden)
    fused.seed_state.set(dev, 4321)
    la = fs.micro_step(ids)
    fused.seed_state.set(dev, 4321)
    lb = ms.micro_step(ids)
    assert abs(float(la) - float(lb)) < 4e-2, (float(la), float(lb))
    ga, gb = _grads(fs), _grads(ms)
    for n in ga:
        if gb[n].norm() == 0:
            continue
        e = _relerr(ga[n], gb[n])
        assert e < 0.15, (n, e)
    before = fs.store.params.clone()
    fs.update()
    assert not torch.equal(before, fs.store.params)
    l2 = fs.micro_step(ids)
    assert torch.isfinite(l2)
    ev = fs.eval_loss(ids)
    assert torch.isfinite(ev) and abs(float(ev) - float(l2)) < 0.5


@pytest.mark.parametrize("shape", [(256, 4, 2), (256, 2, 1)])
def test_native_attention_matches_sdpa_in_the_gqa_executor(shape):
    """The GQA wgmma kernels and torch SDPA (enable_gqa, with rope_pack_bwd gathering nkv-head dk / dv) inside the executor."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    wa = _build(0.1, 512, *shape)
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
    ga, gb = _grads(fa), _grads(fb)
    for n in ga:
        if gb[n].norm() == 0:
            continue
        assert _relerr(ga[n], gb[n]) < 0.1, n


@pytest.mark.parametrize("dx", ["fused", "parts", "base"])
def test_gqa_executor_gemms_match_the_reference(dx, monkeypatch):
    """One training micro-step and one evaluation of the GQA executor with every GEMM and lora_dx call checked against
    ops.reference (the q group and the k | v groups as separate launches into column windows)."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.ops import fused

    C = fused._C()
    if dx == "parts":
        monkeypatch.setenv("RELORA_B200_FUSED_DX", "0")
    if dx == "base":
        monkeypatch.setenv("RELORA_B200_DX_SPLIT_K", "256")
    st = FusedLlamaStepper(_build(0.1, 341), _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False)
    dev = torch.device("cuda", 0)
    ids = torch.randint(0, 1024, (3, 97), device=dev)
    fused.seed_state.set(dev, 4321)
    audit = _Audit(fused, C)
    audit.install(monkeypatch, fused, C)
    loss = st.micro_step(ids)
    ev = st.eval_loss(ids)
    assert torch.isfinite(loss) and torch.isfinite(ev)
    print(f"[gemm modes] audit gqa {dx}: {audit.calls} calls, worst ratio {audit.worst:.3g}, modes {sorted(audit.modes)}")
    want = {"fused": _GROUPED | {"lora_dx"}, "parts": _GROUPED, "base": _GROUPED | {"lora_dx_base"}}[dx]
    assert audit.modes == want


@pytest.mark.parametrize("inter", [512, 341])
def test_fused_gqa_merge_and_checkpoint_roundtrip(tmp_path, inter):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.relora import ReLoRaModel

    w = _build(0.1, inter)
    fs = FusedLlamaStepper(w, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False)
    ids = torch.randint(0, 4096, (2, 64), device="cuda")
    fs.micro_step(ids)
    fs.update()
    w.eval()
    before = fs.eval_loss(ids)
    at = w.wrapped_model.model.layers[0].self_attn
    want = {n: (m.weight.float() + m.scaling * m.lora_B.weight.float() @ m.lora_A.weight.float())
            for n, m in (("q", at.q_proj), ("k", at.k_proj), ("v", at.v_proj))}
    fs.merge_and_reinit()
    for n, m in (("q", at.q_proj), ("k", at.k_proj), ("v", at.v_proj)):
        assert _relerr(m.weight, want[n]) < 4e-3, n
        assert float(m.lora_B.weight.abs().sum()) == 0
    assert at.k_proj.weight.shape == (128, 256) and at.k_proj.weight.data_ptr() == fs.Wqkv[0, 256:384].data_ptr()
    after = fs.eval_loss(ids)
    assert abs(float(before) - float(after)) < 3e-2
    d = str(tmp_path / "m")
    w.save_pretrained(d)
    w2 = ReLoRaModel.from_pretrained(d)
    sd = w.wrapped_model.state_dict()
    for k, v in w2.wrapped_model.state_dict().items():
        assert torch.equal(v.cpu(), sd[k].cpu()), k


def test_cli_end_to_end_from_a_transformers_gqa_checkpoint(tmp_path):
    """torchrun_main --model_name_or_path DIR (a Hugging Face format GQA checkpoint) on the fused executor: a ReLoRA restart,
    finite loss, a checkpoint transformers reads with equal logits, and autoresume."""
    transformers = pytest.importorskip("transformers")
    from relora_b200.models import LlamaForCausalLM, load_config
    from relora_b200.models.llama import load_state_dict_files
    from torchrun_main import main

    ck = tmp_path / "tiny_gqa"
    hcfg = transformers.LlamaConfig(vocab_size=4096, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                                    num_key_value_heads=2, rope_theta=500000.0, max_position_embeddings=256, rms_norm_eps=1e-6,
                                    tie_word_embeddings=False)
    torch.manual_seed(0)
    transformers.LlamaForCausalLM(hcfg).save_pretrained(ck)
    d = str(tmp_path / "run")

    def args(steps, *extra):
        return ["--model_name_or_path", str(ck), "--synthetic_data", "4096", "--batch_size", "4", "--total_batch_size", "8",
                "--max_length", "128", "--lr", "1e-3", "--use_peft", "--lora_r", "128", "--relora", "4", "--cycle_length", "4",
                "--restart_warmup_steps", "1", "--scheduler", "cosine_restarts", "--warmup_steps", "2",
                "--num_training_steps", str(steps), "--save_every", "4", "--eval_every", "100", "--save_dir", d,
                "--dtype", "bfloat16", "--workers", "0", "--init_lora_a", "kaiming", *extra]

    res = main(args(8))
    assert res["executor"] == "FusedLlamaStepper" and res["update_step"] == 8
    assert res["n_lora_restarts"] == 1
    assert torch.isfinite(torch.tensor(res["final_eval_loss"]))
    saved = os.path.join(d, "model_8")
    assert json.load(open(os.path.join(saved, "config.json")))["num_key_value_heads"] == 2
    hf = transformers.LlamaForCausalLM.from_pretrained(saved, attn_implementation="eager").float().eval()
    # the ReLoRA checkpoint also carries the lora_A / lora_B factors, which transformers skips: compare on the frozen weights
    state = {k: v for k, v in load_state_dict_files(saved).items() if "lora_" not in k}
    ours = LlamaForCausalLM(load_config(saved)).float().eval()
    missing, unexpected = ours.load_state_dict(state, strict=False)
    assert not unexpected and all(k.endswith("rotary_emb.inv_freq") for k in missing), (missing, unexpected)
    ids = torch.randint(0, 4096, (2, 33))
    with torch.no_grad():
        assert torch.allclose(hf(input_ids=ids).logits, ours(input_ids=ids).logits, atol=1e-4, rtol=1e-3)
    res2 = main(args(12, "--autoresume", "true"))
    assert res2["update_step"] == 12 and "model_12" in os.listdir(d)
