"""Full-rank selection of the Pythia executor (no GPU): `supports_full_rank()` names the reason for every model it declines and checks
the device last, and the ReLoRA `supports()` answers as before."""
from argparse import Namespace

import pytest
import torch


def _cfg(**over):
    from relora_b200.models import SimpleConfig

    kw = dict(model_type="gpt_neox", vocab_size=256, hidden_size=128, num_hidden_layers=1, num_attention_heads=2, intermediate_size=512,
              rotary_pct=0.25, max_position_embeddings=64, layer_norm_eps=1e-5, use_parallel_residual=True, hidden_act="gelu")
    kw.update(over)
    return SimpleConfig(**kw)


def _neox(**over):
    """A GPT-NeoX on the meta device: the checks read shapes and module types only, so sizes up to the refusal limits cost
    nothing."""
    from relora_b200.models import GPTNeoXForCausalLM

    with torch.device("meta"):
        return GPTNeoXForCausalLM(_cfg(**over)).to(torch.bfloat16)


@pytest.mark.parametrize("over,why", [
    (dict(hidden_dropout=0.1), "dropout must be 0"),
    (dict(attention_dropout=0.1), "dropout must be 0"),
    (dict(hidden_act="relu"), "GELU"),
    (dict(hidden_size=192, num_attention_heads=3, intermediate_size=768), "hidden (192) and intermediate (768) must be multiples of 128"),
    (dict(intermediate_size=320), "hidden (128) and intermediate (320) must be multiples of 128"),
    (dict(hidden_size=2304, num_attention_heads=18, intermediate_size=9216, vocab_size=8), "<= 2048"),
    (dict(num_attention_heads=32), "head_dim (4) must be a multiple of 8"),
    (dict(rotary_pct=0.11), "rotary dims must be even"),
    (dict(attention_bias=False), "projections without bias"),
])
def test_full_rank_names_the_shape_reason(over, why):
    from relora_b200.engine.fused_pythia import supports_full_rank

    ok, reason = supports_full_rank(_neox(**over))
    assert not ok and why in reason, reason


def test_full_rank_refuses_a_projection_without_bias():
    from relora_b200.engine.fused_pythia import supports_full_rank

    m = _neox()
    m.gpt_neox.layers[0].mlp.dense_4h_to_h.bias = None
    assert supports_full_rank(m) == (False, "projections without bias use the module path")


def test_full_rank_refuses_native_attention_above_its_head_dim():
    from relora_b200.engine.fused_pythia import supports_full_rank

    m = _neox(hidden_size=512, num_attention_heads=1, intermediate_size=512)  # head_dim 512
    ok, reason = supports_full_rank(m, Namespace(attention="native"))
    assert not ok and "--attention native supports head_dim <= 256, got 512" in reason
    assert supports_full_rank(m, Namespace(attention="sdpa")) == (False, "needs CUDA + bfloat16")
    assert supports_full_rank(m, Namespace(attention="auto")) == (False, "needs CUDA + bfloat16")


def test_full_rank_refuses_fp8_frozen_weights():
    from relora_b200.engine.fused_pythia import supports_full_rank

    m = _neox()
    for dt in ("fp8", "fp8_full"):
        ok, reason = supports_full_rank(m, Namespace(frozen_dtype=dt))
        assert not ok and f"--frozen_dtype {dt}" in reason and "no frozen weights" in reason


def test_full_rank_checks_the_model_kind_and_the_device_last():
    from relora_b200.engine.fused_pythia import supports_full_rank
    from relora_b200.models import GPTNeoXForCausalLM, LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cpu = GPTNeoXForCausalLM(_cfg()).to(torch.bfloat16)
    assert supports_full_rank(cpu) == (False, "needs CUDA + bfloat16")
    assert supports_full_rank(cpu.float()) == (False, "needs CUDA + bfloat16")
    assert supports_full_rank(_neox(use_parallel_residual=False, hidden_act="gelu_new")) == (False, "needs CUDA + bfloat16")
    # head_dim 256 and a rotary fraction: accepted shapes, native attention included
    assert supports_full_rank(_neox(hidden_size=512, num_attention_heads=2, rotary_pct=0.5), Namespace(attention="native")) == (
        False, "needs CUDA + bfloat16")
    wrapped = ReLoRaModel(GPTNeoXForCausalLM(_cfg()), r=128, lora_alpha=32, lora_dropout=0.0,
                          target_modules=["attn", "attention", "mlp"])
    assert supports_full_rank(wrapped) == (False, "only GPT-NeoX (Pythia) is fused for full-rank training here")
    llama = LlamaForCausalLM(SimpleConfig(model_type="llama", vocab_size=256, hidden_size=256, intermediate_size=512,
                                          num_hidden_layers=1, num_attention_heads=4, rms_norm_eps=1e-6, pad_token_id=-1,
                                          max_position_embeddings=64))
    assert supports_full_rank(llama) == (False, "only GPT-NeoX (Pythia) is fused for full-rank training here")


def test_relora_supports_is_unchanged():
    """The ReLoRA `supports()` gives its previous answers for a bare model, a wrapped model and a CPU model."""
    from relora_b200.engine.fused_pythia import supports
    from relora_b200.models import GPTNeoXForCausalLM
    from relora_b200.relora import ReLoRaModel

    def wrap(r=128, **over):
        return ReLoRaModel(GPTNeoXForCausalLM(_cfg(**over)), r=r, lora_alpha=32, lora_dropout=0.1,
                           target_modules=["attn", "attention", "mlp"]).to(torch.bfloat16)

    bare = GPTNeoXForCausalLM(_cfg()).to(torch.bfloat16)
    assert supports(bare) == (False, "full-rank training uses the module path")
    m = wrap()
    assert supports(m.wrapped_model) == (False, "full-rank training uses the module path")
    assert supports(m) == (False, "needs CUDA + bfloat16")
    assert supports(m, Namespace(frozen_dtype="fp8")) == (False, "fp8 frozen weights are not supported for Pythia")
    assert supports(wrap(r=64)) == (False, "hidden (128), intermediate (512) and rank (64) must be multiples of 128")
