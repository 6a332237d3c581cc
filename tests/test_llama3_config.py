"""Llama-3.1's ``llama3`` rotary scaling on CPU: the config is accepted in both dialects (``rope_scaling`` and transformers >= 5's
``rope_parameters``) and refused by name when a setting is missing, ``inv_freq`` and logits agree with transformers, the layers
share one rotary table, and the CLI trains from such a checkpoint and saves one transformers reloads with the same settings."""
import json
import os

import pytest
import torch

transformers = pytest.importorskip("transformers")

# head_dim 64, θ 10000 and an original context of 32 positions: 31 of the 32 frequencies change (stretched or blended)
LLAMA3 = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 32}
KEYS = ("factor", "low_freq_factor", "high_freq_factor", "original_max_position_embeddings")


def _raw(**kw):
    raw = dict(model_type="llama", vocab_size=97, hidden_size=256, intermediate_size=96, num_hidden_layers=3, num_attention_heads=4,
               num_key_value_heads=2, rope_theta=10000.0, max_position_embeddings=128, rms_norm_eps=1e-6, tie_word_embeddings=False)
    raw.update(kw)
    return raw


def _dialect(name, scaling):
    if name == "rope_scaling":
        return dict(rope_scaling=dict(scaling))
    return dict(rope_parameters=dict(scaling, rope_theta=10000.0))


def _hf_cfg(**kw):
    raw = _raw(rope_scaling=dict(LLAMA3), **kw)
    raw.pop("model_type")
    return transformers.LlamaConfig(**raw)


def _unscaled(dim=64, theta=10000.0):
    return 1.0 / (theta ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim))


@pytest.mark.parametrize("dialect", ["rope_scaling", "rope_parameters"])
def test_llama3_is_accepted_in_both_dialects(dialect):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.models.llama import llama3_rope_parameters

    cfg = SimpleConfig(**_raw(**_dialect(dialect, LLAMA3)))
    assert llama3_rope_parameters(cfg) == {k: float(LLAMA3[k]) for k in KEYS}
    inv = LlamaForCausalLM(cfg).model.layers[0].self_attn.rotary_emb.inv_freq
    hf = transformers.LlamaForCausalLM(_hf_cfg()).model.rotary_emb.inv_freq
    assert torch.equal(inv, hf)


@pytest.mark.parametrize("dialect", ["rope_scaling", "rope_parameters"])
@pytest.mark.parametrize("key", KEYS)
def test_llama3_missing_setting_is_refused_by_name(tmp_path, dialect, key):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig

    scaling = {k: v for k, v in LLAMA3.items() if k != key}
    raw = _raw(**_dialect(dialect, scaling))
    with pytest.raises(ValueError, match=key):
        LlamaForCausalLM(SimpleConfig(**raw))
    with open(tmp_path / "config.json", "w") as f:
        json.dump(raw, f)
    if key == "original_max_position_embeddings":
        # transformers reads a config.json without it as original_max_position_embeddings = max_position_embeddings; the
        # model built from that file follows the same reading
        from relora_b200.models import load_config

        cfg = load_config(str(tmp_path))
        hf = transformers.LlamaForCausalLM(cfg).model.rotary_emb.inv_freq
        assert torch.equal(LlamaForCausalLM(cfg).model.layers[0].self_attn.rotary_emb.inv_freq, hf)
        return
    torch.save({}, tmp_path / "pytorch_model.bin")
    with pytest.raises(ValueError, match=key):
        LlamaForCausalLM.from_pretrained(str(tmp_path))


@pytest.mark.parametrize("dialect", ["rope_scaling", "rope_parameters"])
@pytest.mark.parametrize("kind", ["linear", "dynamic", "yarn", "longrope"])
def test_other_scaling_types_are_still_refused(dialect, kind):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig

    with pytest.raises(ValueError, match="rope_scaling"):
        LlamaForCausalLM(SimpleConfig(**_raw(**_dialect(dialect, {"rope_type": kind, "factor": 2.0}))))


def test_inv_freq_equals_transformers_and_differs_from_unscaled():
    from relora_b200.models import LlamaForCausalLM

    cfg = _hf_cfg()
    want = transformers.LlamaForCausalLM(cfg).model.rotary_emb.inv_freq
    got = LlamaForCausalLM(cfg).model.layers[0].self_attn.rotary_emb.inv_freq
    assert got.dtype == torch.float32 and torch.equal(got, want)
    unscaled = _unscaled()
    assert int((got != unscaled).sum()) >= 30
    # the lowest frequencies are stretched by the full factor, the highest one is kept
    assert torch.allclose(got[-1], unscaled[-1] / 8.0) and torch.equal(got[0], unscaled[0])


def _save_hf(d, seed=0, **kw):
    torch.manual_seed(seed)
    cfg = _hf_cfg(**kw)
    cfg._attn_implementation = "eager"
    hf = transformers.LlamaForCausalLM(cfg).float().eval()
    hf.save_pretrained(d)
    return hf


def test_logits_match_transformers_from_the_same_checkpoint(tmp_path):
    from relora_b200.models import LlamaForCausalLM

    _save_hf(tmp_path)
    hf = transformers.LlamaForCausalLM.from_pretrained(str(tmp_path), attn_implementation="eager").float().eval()
    ours = LlamaForCausalLM.from_pretrained(str(tmp_path)).float().eval()
    ids = torch.randint(0, 97, (2, 64), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want, got = hf(input_ids=ids).logits, ours(input_ids=ids).logits
    assert torch.allclose(got, want, atol=1e-5, rtol=1e-4)
    # the scaling matters at these positions: the unscaled model gives other logits
    plain = LlamaForCausalLM.from_pretrained(str(tmp_path)).float().eval()
    for layer in plain.model.layers:
        layer.self_attn.rotary_emb._build(128, _unscaled())
    with torch.no_grad():
        assert not torch.allclose(plain(input_ids=ids).logits, want, atol=1e-3)


def test_layers_share_one_rotary_table():
    from relora_b200.models import LlamaForCausalLM

    model = LlamaForCausalLM(_hf_cfg())
    rots = [layer.self_attn.rotary_emb for layer in model.model.layers]
    assert all(r is rots[0] for r in rots)
    model = model.to(torch.bfloat16)
    rots = [layer.self_attn.rotary_emb for layer in model.model.layers]
    assert len({r.cos_cached.data_ptr() for r in rots}) == 1 and rots[0].cos_cached.dtype == torch.bfloat16
    # the state dict still names inv_freq under every layer, as reference checkpoints do; the tables are not saved
    keys = model.state_dict().keys()
    assert all(f"model.layers.{i}.self_attn.rotary_emb.inv_freq" in keys for i in range(3))
    assert not any("cos_cached" in k or "sin_cached" in k for k in keys)


def test_cli_trains_relora_from_a_llama3_checkpoint(tmp_path):
    from torchrun_main import main

    ck = tmp_path / "tiny_llama3"
    _save_hf(ck, vocab_size=32100)
    d = str(tmp_path / "run")
    res = main(["--model_name_or_path", str(ck), "--synthetic_data", "2048", "--batch_size", "2", "--total_batch_size", "4",
                "--max_length", "64", "--lr", "1e-3", "--use_peft", "--lora_r", "4", "--relora", "4", "--cycle_length", "4",
                "--restart_warmup_steps", "1", "--scheduler", "cosine_restarts", "--warmup_steps", "2", "--num_training_steps", "8",
                "--save_every", "8", "--eval_every", "100", "--save_dir", d, "--device", "cpu", "--dtype", "float32", "--workers", "0"])
    assert res["update_step"] == 8 and res["n_lora_restarts"] == 1
    assert res["final_eval_loss"] == res["final_eval_loss"]
    saved = transformers.LlamaForCausalLM.from_pretrained(os.path.join(d, "model_8"), attn_implementation="eager").float()
    rp = saved.config.rope_parameters
    assert {k: rp[k] for k in ("rope_type", *KEYS)} == LLAMA3 and rp["rope_theta"] == 10000.0
    want = transformers.LlamaForCausalLM(_hf_cfg()).model.rotary_emb.inv_freq
    assert torch.equal(saved.model.rotary_emb.inv_freq, want)
