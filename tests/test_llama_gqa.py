"""Grouped-query attention and ``rope_theta`` for Llama-family models on CPU: parity with ``transformers.LlamaForCausalLM``,
checkpoint round trips in both directions, the refused config options, and a short CLI run from a local checkpoint."""
import json
import os

import pytest
import torch

transformers = pytest.importorskip("transformers")


def _cfg(nkv, rope_theta=10000.0, **kw):
    base = dict(vocab_size=97, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=4,
                num_key_value_heads=nkv, rope_theta=rope_theta, max_position_embeddings=64, rms_norm_eps=1e-6,
                tie_word_embeddings=False)
    base.update(kw)
    return transformers.LlamaConfig(**base)


def _hf(cfg, seed=0):
    torch.manual_seed(seed)
    cfg._attn_implementation = "eager"
    return transformers.LlamaForCausalLM(cfg).float().eval()


def _ours_from(hf):
    from relora_b200.models import LlamaForCausalLM

    ours = LlamaForCausalLM(hf.config).float().eval()
    missing, unexpected = ours.load_state_dict(hf.state_dict(), strict=False)
    assert not unexpected and all(k.endswith("rotary_emb.inv_freq") for k in missing), (missing, unexpected)
    return ours


@pytest.mark.parametrize("nkv", [1, 2, 4])
@pytest.mark.parametrize("rope_theta", [10000.0, 500000.0])
def test_gqa_matches_transformers_logits_and_grads(nkv, rope_theta):
    hf = _hf(_cfg(nkv, rope_theta))
    ours = _ours_from(hf)
    at = ours.model.layers[0].self_attn
    assert at.k_proj.weight.shape == (nkv * 16, 64) and at.num_key_value_groups == 4 // nkv
    assert torch.allclose(at.rotary_emb.inv_freq, 1.0 / rope_theta ** (torch.arange(0, 16, 2).float() / 16))
    ids = torch.randint(0, 97, (2, 23), generator=torch.Generator().manual_seed(1))
    out_hf = hf(input_ids=ids, labels=ids)
    out = ours(input_ids=ids, labels=ids)
    assert torch.allclose(out.logits, out_hf.logits, atol=1e-5, rtol=1e-4)
    out_hf.loss.backward()
    out.loss.backward()
    ref = dict(hf.named_parameters())
    for n, p in ours.named_parameters():
        assert torch.allclose(p.grad, ref[n].grad, atol=1e-6, rtol=1e-4), n


def test_gqa_kv_cache_generation_matches_full_forward():
    ours = _ours_from(_hf(_cfg(2)))
    ids = torch.randint(0, 97, (1, 7), generator=torch.Generator().manual_seed(2))
    toks = ours.generate(ids, max_new_tokens=5)
    full = ours(input_ids=toks[:, :-1]).logits
    assert torch.equal(full[:, 6:].argmax(-1), toks[:, 7:])


def _save_hf(hf, d, **kw):
    hf.save_pretrained(d, **kw)
    return sorted(os.listdir(d))


@pytest.mark.parametrize("sharded", [False, True])
def test_transformers_safetensors_checkpoint_loads(tmp_path, sharded):
    from relora_b200.models import LlamaForCausalLM

    hf = _hf(_cfg(2, 500000.0))
    files = _save_hf(hf, tmp_path, max_shard_size="20KB" if sharded else "5GB")
    assert ("model.safetensors.index.json" in files) == sharded
    ours = LlamaForCausalLM.from_pretrained(str(tmp_path)).eval()
    assert ours.model.layers[0].self_attn.rotary_emb.base == 500000.0
    ids = torch.randint(0, 97, (2, 11))
    assert torch.allclose(ours(input_ids=ids).logits, hf(input_ids=ids).logits, atol=1e-5, rtol=1e-4)


def test_bin_checkpoint_and_sharded_bin_index_load(tmp_path):
    from relora_b200.models import LlamaForCausalLM

    hf = _hf(_cfg(1))
    hf.config.save_pretrained(tmp_path / "single")
    state = {k: v.clone() for k, v in hf.state_dict().items()}
    torch.save(state, tmp_path / "single" / "pytorch_model.bin")
    hf.config.save_pretrained(tmp_path / "sharded")
    keys = sorted(state)
    halves = {"pytorch_model-00001-of-00002.bin": keys[: len(keys) // 2], "pytorch_model-00002-of-00002.bin": keys[len(keys) // 2:]}
    weight_map = {}
    for fname, ks in halves.items():
        torch.save({k: state[k] for k in ks}, tmp_path / "sharded" / fname)
        weight_map.update({k: fname for k in ks})
    with open(tmp_path / "sharded" / "pytorch_model.bin.index.json", "w") as f:
        json.dump({"metadata": {}, "weight_map": weight_map}, f)
    ids = torch.randint(0, 97, (1, 9))
    want = hf(input_ids=ids).logits
    for sub in ("single", "sharded"):
        ours = LlamaForCausalLM.from_pretrained(str(tmp_path / sub)).eval()
        assert torch.allclose(ours(input_ids=ids).logits, want, atol=1e-5, rtol=1e-4), sub


def test_missing_or_unexpected_key_is_an_error(tmp_path):
    from relora_b200.models import LlamaForCausalLM

    hf = _hf(_cfg(2))
    hf.config.save_pretrained(tmp_path)
    state = dict(hf.state_dict())
    state.pop("model.layers.1.mlp.up_proj.weight")
    torch.save(state, tmp_path / "pytorch_model.bin")
    with pytest.raises(RuntimeError, match="up_proj"):
        LlamaForCausalLM.from_pretrained(str(tmp_path))
    state = dict(hf.state_dict())
    state["model.layers.0.self_attn.q_proj.bias"] = torch.zeros(64)
    torch.save(state, tmp_path / "pytorch_model.bin")
    with pytest.raises(RuntimeError, match="q_proj.bias"):
        LlamaForCausalLM.from_pretrained(str(tmp_path))


def test_our_checkpoint_loads_into_transformers(tmp_path):
    from relora_b200.models import LlamaForCausalLM, load_config

    cfg = _cfg(2, 500000.0)
    torch.manual_seed(3)
    ours = LlamaForCausalLM(cfg).float().eval()
    ours.save_pretrained(str(tmp_path))
    saved = json.load(open(tmp_path / "config.json"))
    assert saved["num_key_value_heads"] == 2
    assert load_config(str(tmp_path)).num_key_value_heads == 2
    theta = saved.get("rope_theta", (saved.get("rope_parameters") or {}).get("rope_theta"))
    assert theta == 500000.0
    hf = transformers.LlamaForCausalLM.from_pretrained(str(tmp_path), attn_implementation="eager").float().eval()
    ids = torch.randint(0, 97, (2, 13))
    assert torch.allclose(hf(input_ids=ids).logits, ours(input_ids=ids).logits, atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("field,kw", [
    ("rope_scaling", dict(rope_scaling={"rope_type": "linear", "factor": 2.0})),
    ("tie_word_embeddings", dict(tie_word_embeddings=True)),
    ("attention_bias", dict(attention_bias=True)),
    ("mlp_bias", dict(mlp_bias=True)),
    ("head_dim", dict(head_dim=32)),
    ("num_key_value_heads", dict(num_key_value_heads=3)),
])
def test_unsupported_config_fields_are_refused(tmp_path, field, kw):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig

    raw = dict(model_type="llama", vocab_size=97, hidden_size=64, intermediate_size=96, num_hidden_layers=1,
               num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=64)
    raw.update(kw)
    with pytest.raises(ValueError, match=field):
        LlamaForCausalLM(SimpleConfig(**raw))
    # the same refusal when a checkpoint directory carries the field
    with open(tmp_path / "config.json", "w") as f:
        json.dump(raw, f)
    torch.save({}, tmp_path / "pytorch_model.bin")
    with pytest.raises(ValueError, match=field):
        LlamaForCausalLM.from_pretrained(str(tmp_path))


def test_fused_executor_gqa_supports_reasons():
    """The executor takes GQA when nkv x head_dim is a multiple of 128 and declines it, naming the reason, otherwise and with
    the fp8 frozen-weight path (on CPU every model then stops at the CUDA requirement)."""
    import argparse

    from relora_b200.engine.fused_llama import supports
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    def wrap(nkv):
        cfg = SimpleConfig(model_type="llama", vocab_size=97, hidden_size=256, intermediate_size=256, num_hidden_layers=1,
                           num_attention_heads=4, num_key_value_heads=nkv, max_position_embeddings=64)
        return ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "mlp"])

    ok, why = supports(wrap(1))
    assert not ok and "num_key_value_heads x head_dim (1 x 64)" in why
    ok, why = supports(wrap(2), argparse.Namespace(frozen_dtype="fp8"))
    assert not ok and "fp8" in why and "grouped-query" in why
    ok, why = supports(wrap(2))
    assert not ok and why == "needs CUDA + bfloat16"


def test_warmed_up_model_from_a_transformers_gqa_checkpoint(tmp_path):
    """--warmed_up_model reads the same checkpoint forms as --model_name_or_path (sharded safetensors, no inv_freq)."""
    from relora_b200.ckpt import load_model_weights
    from relora_b200.models import LlamaForCausalLM, load_config
    from torchrun_main import main

    ck = tmp_path / "warm"
    hf = _hf(_cfg(2, 500000.0, vocab_size=32100))
    hf.save_pretrained(ck, max_shard_size="200KB")
    assert (ck / "model.safetensors.index.json").exists()
    ours = LlamaForCausalLM(load_config(str(ck))).float().eval()
    load_model_weights(ours, str(ck))
    ids = torch.randint(0, 97, (1, 9))
    assert torch.allclose(ours(input_ids=ids).logits, hf(input_ids=ids).logits, atol=1e-5, rtol=1e-4)
    res = main(["--model_config", str(ck / "config.json"), "--warmed_up_model", str(ck), "--synthetic_data", "1024",
                "--batch_size", "2", "--total_batch_size", "2", "--max_length", "32", "--lr", "1e-3", "--use_peft", "--lora_r", "4",
                "--relora", "2", "--cycle_length", "2", "--restart_warmup_steps", "1", "--scheduler", "cosine_restarts",
                "--warmup_steps", "1", "--num_training_steps", "4", "--save_every", "4", "--eval_every", "100",
                "--save_dir", str(tmp_path / "run"), "--device", "cpu", "--dtype", "float32", "--workers", "0"])
    assert res["update_step"] == 4 and res["final_eval_loss"] == res["final_eval_loss"]


def test_simple_config_carries_kv_heads_and_rope_theta(tmp_path):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig

    LlamaForCausalLM(SimpleConfig(model_type="llama", vocab_size=97, hidden_size=64, intermediate_size=96, num_hidden_layers=1,
                                  num_attention_heads=4, max_position_embeddings=64)).save_pretrained(str(tmp_path))
    saved = json.load(open(tmp_path / "config.json"))
    assert saved.get("num_key_value_heads") == 4
    assert (saved.get("rope_theta") or (saved.get("rope_parameters") or {}).get("rope_theta")) == 10000.0


def test_cli_trains_from_a_local_gqa_checkpoint(tmp_path):
    from torchrun_main import main

    ck = tmp_path / "tiny_gqa"
    hf = _hf(_cfg(2, 500000.0, vocab_size=32100, max_position_embeddings=64))
    hf.save_pretrained(ck)
    d = str(tmp_path / "run")

    def args(steps, *extra):
        return ["--model_name_or_path", str(ck), "--synthetic_data", "2048", "--batch_size", "2", "--total_batch_size", "4",
                "--max_length", "32", "--lr", "1e-3", "--use_peft", "--lora_r", "4", "--relora", "4", "--cycle_length", "4",
                "--restart_warmup_steps", "1", "--scheduler", "cosine_restarts", "--warmup_steps", "2",
                "--num_training_steps", str(steps), "--save_every", "4", "--eval_every", "100", "--save_dir", d,
                "--device", "cpu", "--dtype", "float32", "--workers", "0", *extra]

    res = main(args(8))
    assert res["update_step"] == 8 and res["n_lora_restarts"] == 1 and res["executor"] == "ModuleStepper"
    assert res["final_eval_loss"] == res["final_eval_loss"]
    saved = transformers.LlamaForCausalLM.from_pretrained(os.path.join(d, "model_8"), attn_implementation="eager").float()
    assert saved.config.num_key_value_heads == 2
    assert saved.model.layers[0].self_attn.k_proj.weight.shape == (32, 64)
    res2 = main(args(12, "--autoresume", "true"))
    assert res2["update_step"] == 12
