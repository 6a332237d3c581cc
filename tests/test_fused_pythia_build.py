"""Build-time facts of the Pythia executor (no GPU): its kernels compile without spills, and `supports()` names the reason for every
configuration it declines."""
import importlib
import os
import re

import pytest
import torch

NEW_KERNELS = ("layernorm_fwd_kernel", "layernorm_bwd_dual_kernel", "gelu_fwd_kernel", "colsum_kernel", "attn_fwd_kernel",
               "attn_bwd_dq_kernel", "attn_bwd_dkv_kernel")


def test_executor_kernels_compile_without_spills():
    build = importlib.import_module("relora_b200.csrc.build")
    if not os.path.exists(os.path.join(build.BUILD_DIR, "neox.cu.log")):
        pytest.skip("needs the built extension")
    seen, cur = {}, None
    for line in build.ptxas_report().splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = next((k + m.group(1)[-40:] for k in NEW_KERNELS if k in m.group(1)), None)
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur:
            seen[cur] = int(m.group(1))
            cur = None
    for k in NEW_KERNELS:
        assert any(n.startswith(k) for n in seen), (k, sorted(seen))
    assert all(v == 0 for v in seen.values()), {k: v for k, v in seen.items() if v}


def _model(**over):
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    kw = dict(model_type="gpt_neox", vocab_size=256, hidden_size=128, num_hidden_layers=1, num_attention_heads=2, intermediate_size=512,
              rotary_pct=0.25, max_position_embeddings=64, layer_norm_eps=1e-5, use_parallel_residual=True, hidden_act="gelu")
    relora = {k: over.pop(k) for k in ("r", "lora_only", "trainable_scaling") if k in over}
    kw.update(over)
    return ReLoRaModel(GPTNeoXForCausalLM(SimpleConfig(**kw)), r=relora.get("r", 128), lora_alpha=32, lora_dropout=0.1,
                       target_modules=["attn", "attention", "mlp"], lora_only=relora.get("lora_only", False),
                       trainable_scaling=relora.get("trainable_scaling", False)).to(torch.bfloat16)


@pytest.mark.parametrize("over,why", [
    (dict(lora_only=True), "lora_only"),
    (dict(trainable_scaling=True), "trainable scaling"),
    (dict(hidden_dropout=0.1), "dropout"),
    (dict(attention_dropout=0.1), "dropout"),
    (dict(hidden_act="relu"), "GELU"),
    (dict(r=64), "multiples of 128"),
    (dict(hidden_size=192, num_attention_heads=3, intermediate_size=768), "multiples of 128"),
    (dict(hidden_size=2304, num_attention_heads=18, intermediate_size=9216), "<= 2048"),
    (dict(num_attention_heads=32), "head_dim"),
    (dict(rotary_pct=0.11), "rotary"),
    (dict(attention_bias=False), "bias"),
])
def test_supports_names_the_reason(over, why):
    from relora_b200.engine.fused_pythia import supports

    ok, reason = supports(_model(**over))
    assert not ok and why in reason, reason


def test_supports_checks_the_recipe_flags_and_the_device_last():
    from argparse import Namespace

    from relora_b200.engine.fused_pythia import supports

    m = _model()
    assert supports(m, Namespace(frozen_dtype="fp8")) == (False, "fp8 frozen weights are not supported for Pythia")
    assert supports(m) == (False, "needs CUDA + bfloat16")  # the model is on the CPU here
    assert supports(m.wrapped_model)[0] is False
