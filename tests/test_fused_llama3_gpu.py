"""A Llama-3-shaped model on the H100 (-m gpu): a 128,256-token vocabulary, whose cross-entropy takes the streaming kernel, and
llama3 rotary scaling.  The fused executor against the module path on identical weights and dropout masks (ReLoRA and full-rank),
the module path on CUDA against the fp32 CPU loss, and the CLI end to end from a transformers checkpoint."""
import copy
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
VOCAB = 128256
LLAMA3 = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 64}


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


def _cfg():
    from relora_b200.models import SimpleConfig

    return SimpleConfig(model_type="llama", vocab_size=VOCAB, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                        num_attention_heads=4, num_key_value_heads=2, rope_theta=500000.0, rms_norm_eps=1e-6, pad_token_id=-1,
                        max_position_embeddings=256, rope_scaling=dict(LLAMA3))


def _llama(seed=0):
    from relora_b200.models import LlamaForCausalLM

    torch.manual_seed(seed)
    return LlamaForCausalLM(_cfg())


def _relora(p_drop):
    from relora_b200.relora import ReLoRaModel

    w = ReLoRaModel(_llama(), r=128, lora_alpha=32, lora_dropout=p_drop, target_modules=["attn", "mlp"], init_lora_a="kaiming")
    torch.manual_seed(1)
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _grads(st):
    return {n: st.store.view_like(st.store.grads, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


def _ids(B=3, T=128):
    return torch.randint(0, VOCAB, (B, T), generator=torch.Generator().manual_seed(5)).cuda()


def _compare(fs, ms):
    dev = torch.device("cuda", 0)
    from relora_b200.ops import fused

    ids = _ids()
    fused.seed_state.set(dev, 4321)
    la = fs.micro_step(ids)
    fused.seed_state.set(dev, 4321)
    lb = ms.micro_step(ids)
    assert abs(float(la) - float(lb)) < 4e-2, (float(la), float(lb))
    ga, gb = _grads(fs), _grads(ms)
    assert any(n.endswith("lm_head.weight") for n in ga)
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


@pytest.mark.parametrize("p_drop,graphs", [(0.0, False), (0.1, False), (0.0, True), (0.1, True)])
def test_fused_relora_matches_module_path(p_drop, graphs):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    wa = _relora(p_drop)
    wb = copy.deepcopy(wa)
    fs = FusedLlamaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs)
    ms = ModuleStepper(wb, _info(), lr=1e-3, grad_accumulation=1, native=fused.NativeOptim())
    assert fs.V == VOCAB
    # the executor's rotary tables are the llama3-scaled ones of the model
    rot = wa.wrapped_model.model.layers[0].self_attn.rotary_emb
    assert rot.llama3 is not None and torch.equal(fs.cos, rot.cos_cached[0, 0].to(BF))
    _compare(fs, ms)


@pytest.mark.parametrize("graphs", [False, True])
def test_fused_full_rank_matches_module_path(graphs):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    ma = _llama().cuda().to(BF)
    mb = copy.deepcopy(ma)
    fs = FusedLlamaStepper(ma, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs)
    ms = ModuleStepper(mb, _info(), lr=1e-3, grad_accumulation=1, native=fused.NativeOptim())
    _compare(fs, ms)


def test_module_path_on_cuda_matches_the_fp32_cpu_loss():
    """bf16 on CUDA, with the chunked LM head + streaming cross-entropy (return_logits=False) and with full logits, against the
    fp32 model on the CPU."""
    cpu = _llama().float()
    gpu = copy.deepcopy(cpu).cuda().to(BF)
    ids = _ids(2, 128)
    want = cpu(input_ids=ids.cpu(), labels=ids.cpu())
    want.loss.backward()
    got = gpu(input_ids=ids, labels=ids, return_logits=False)
    got.loss.backward()
    full = gpu(input_ids=ids, labels=ids)
    assert abs(float(got.loss) - float(want.loss)) < 2e-2, (float(got.loss), float(want.loss))
    assert abs(float(full.loss) - float(want.loss)) < 2e-2, (float(full.loss), float(want.loss))
    assert _relerr(gpu.lm_head.weight.grad.cpu(), cpu.lm_head.weight.grad) < 0.1
    assert _relerr(gpu.model.embed_tokens.weight.grad.cpu(), cpu.model.embed_tokens.weight.grad) < 0.1


def test_cli_end_to_end_from_a_transformers_llama3_checkpoint(tmp_path):
    """torchrun_main --engine fused from a transformers llama3 checkpoint: a ReLoRA restart (merge), finite loss, and a saved
    checkpoint transformers reads with the same rope settings and equal logits."""
    transformers = pytest.importorskip("transformers")
    from relora_b200.models import LlamaForCausalLM, load_config
    from relora_b200.models.llama import load_state_dict_files
    from torchrun_main import main

    ck = tmp_path / "tiny_llama3"
    hcfg = transformers.LlamaConfig(vocab_size=VOCAB, hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                                    num_key_value_heads=2, rope_theta=500000.0, max_position_embeddings=256, rms_norm_eps=1e-6,
                                    tie_word_embeddings=False, rope_scaling=dict(LLAMA3))
    torch.manual_seed(0)
    transformers.LlamaForCausalLM(hcfg).save_pretrained(ck)
    d = str(tmp_path / "run")
    res = main(["--model_name_or_path", str(ck), "--synthetic_data", "4096", "--batch_size", "4", "--total_batch_size", "8",
                "--max_length", "128", "--lr", "1e-3", "--use_peft", "--lora_r", "128", "--relora", "4", "--cycle_length", "4",
                "--restart_warmup_steps", "1", "--scheduler", "cosine_restarts", "--warmup_steps", "2", "--num_training_steps", "8",
                "--save_every", "8", "--eval_every", "100", "--save_dir", d, "--dtype", "bfloat16", "--workers", "0",
                "--init_lora_a", "kaiming", "--engine", "fused"])
    assert res["executor"] == "FusedLlamaStepper" and res["update_step"] == 8 and res["n_lora_restarts"] == 1
    assert torch.isfinite(torch.tensor(res["final_eval_loss"]))
    saved = os.path.join(d, "model_8")
    rp = json.load(open(os.path.join(saved, "config.json")))
    rp = rp.get("rope_parameters") or rp["rope_scaling"]
    assert {k: rp[k] for k in LLAMA3} == LLAMA3
    hf = transformers.LlamaForCausalLM.from_pretrained(saved, attn_implementation="eager").float().eval()
    state = {k: v for k, v in load_state_dict_files(saved).items() if "lora_" not in k}
    ours = LlamaForCausalLM(load_config(saved)).float().eval()
    # built from the saved config (the checkpoint's own inv_freq buffers are the bf16 copies the run trained with)
    assert torch.equal(ours.model.layers[0].self_attn.rotary_emb.inv_freq, hf.model.rotary_emb.inv_freq)
    missing, unexpected = ours.load_state_dict(state, strict=False)
    assert not unexpected and all(k.endswith("rotary_emb.inv_freq") for k in missing), (missing, unexpected)
    ids = torch.randint(0, VOCAB, (2, 33))
    with torch.no_grad():
        assert torch.allclose(hf(input_ids=ids).logits, ours(input_ids=ids).logits, atol=1e-4, rtol=1e-3)
