"""Full-rank selection of the Llama executor (no GPU): `supports_full_rank()` names the reason for every model it declines and checks
the device last, and the ReLoRA `supports()` answers as before."""
from argparse import Namespace

import pytest
import torch


def _cfg(**over):
    from relora_b200.models import SimpleConfig

    kw = dict(model_type="llama", vocab_size=256, hidden_size=256, intermediate_size=512, num_hidden_layers=1, num_attention_heads=4,
              rms_norm_eps=1e-6, pad_token_id=-1, max_position_embeddings=64)
    kw.update(over)
    return SimpleConfig(**kw)


def _llama(**over):
    """A Llama on the meta device: the checks read shapes and module types only, so sizes up to the refusal limits cost nothing."""
    from relora_b200.models import LlamaForCausalLM

    with torch.device("meta"):
        return LlamaForCausalLM(_cfg(**over)).to(torch.bfloat16)


@pytest.mark.parametrize("over,why", [
    (dict(hidden_size=36, num_attention_heads=4, intermediate_size=64), "16-byte row pitch"),
    (dict(hidden_size=24, num_attention_heads=3, intermediate_size=64), "stacked q | k | v"),
    (dict(hidden_size=8320, num_attention_heads=65, intermediate_size=128, vocab_size=8), "RMSNorm"),
    (dict(hidden_size=96, num_attention_heads=8, intermediate_size=128), "head_dim (12) must be a multiple of 8"),
])
def test_full_rank_names_the_shape_reason(over, why):
    from relora_b200.engine.fused_llama import supports_full_rank

    ok, reason = supports_full_rank(_llama(**over))
    assert not ok and why in reason, reason


def test_full_rank_refuses_native_attention_above_its_head_dim():
    from relora_b200.engine.fused_llama import supports_full_rank

    m = _llama(hidden_size=512, num_attention_heads=1, num_key_value_heads=1)  # head_dim 512
    ok, reason = supports_full_rank(m, Namespace(attention="native"))
    assert not ok and "--attention native supports head_dim <= 256, got 512" in reason
    assert supports_full_rank(m, Namespace(attention="sdpa")) == (False, "needs CUDA + bfloat16")


def test_full_rank_refuses_fp8_frozen_weights_and_biases():
    from relora_b200.engine.fused_llama import supports_full_rank

    m = _llama()
    for dt in ("fp8", "fp8_full"):
        ok, reason = supports_full_rank(m, Namespace(frozen_dtype=dt))
        assert not ok and f"--frozen_dtype {dt}" in reason and "frozen" in reason
    up = m.model.layers[0].mlp.up_proj
    up.bias = torch.nn.Parameter(torch.zeros(up.out_features, device="meta", dtype=torch.bfloat16))
    assert supports_full_rank(m) == (False, "biased projections use the module path")


def test_full_rank_checks_the_model_kind_and_the_device_last():
    from relora_b200.engine.fused_llama import supports_full_rank
    from relora_b200.models import GPTNeoXForCausalLM, LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cpu = LlamaForCausalLM(_cfg(num_key_value_heads=1)).to(torch.bfloat16)  # GQA: k / v 64 wide, q 256
    assert supports_full_rank(cpu) == (False, "needs CUDA + bfloat16")
    assert supports_full_rank(cpu.float()) == (False, "needs CUDA + bfloat16")
    assert supports_full_rank(_llama(intermediate_size=341)) == (False, "needs CUDA + bfloat16")  # padded MLP: accepted shape
    wrapped = ReLoRaModel(LlamaForCausalLM(_cfg()), r=128, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "mlp"])
    assert supports_full_rank(wrapped) == (False, "only Llama is fused for full-rank training")
    neox = GPTNeoXForCausalLM(SimpleConfig(model_type="gpt_neox", vocab_size=256, hidden_size=128, num_hidden_layers=1,
                                           num_attention_heads=2, intermediate_size=512, rotary_pct=0.25, max_position_embeddings=64,
                                           layer_norm_eps=1e-5, use_parallel_residual=True, hidden_act="gelu"))
    assert supports_full_rank(neox) == (False, "only Llama is fused for full-rank training")


def test_relora_supports_is_unchanged():
    from relora_b200.engine.fused_llama import supports
    from relora_b200.models import LlamaForCausalLM
    from relora_b200.relora import ReLoRaModel

    def wrap(r=128, **over):
        return ReLoRaModel(LlamaForCausalLM(_cfg(**over)), r=r, lora_alpha=32, lora_dropout=0.1,
                           target_modules=["attn", "mlp"]).to(torch.bfloat16)

    assert supports(LlamaForCausalLM(_cfg())) == (False, "full-rank training uses the module path")
    assert supports(wrap()) == (False, "needs CUDA + bfloat16")
    assert supports(wrap(r=64)) == (False, "hidden (256) and rank (64) must be multiples of 128 for stacked groups")
    assert supports(wrap(num_attention_heads=8, num_key_value_heads=2)) == (
        False, "grouped-query attention needs num_key_value_heads x head_dim (2 x 32) to be a multiple of 128")
    assert supports(wrap(num_key_value_heads=2), Namespace(frozen_dtype="fp8")) == (
        False, "--frozen_dtype fp8 with grouped-query attention uses the module path (the fp8 weight copies are [3h, h])")
