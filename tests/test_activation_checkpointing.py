"""`--activation_checkpointing` without a GPU: the flag and its place among the engine flags, the module path's per-layer
checkpointing (bit-identical gradients on tiny Llama and Pythia ReLoRA models) and the refusal of the fp8 frozen-weight path."""
import argparse
import copy

import pytest
import torch
import yaml

from relora_b200.config import ENGINE_FLAGS, parse_args
from relora_b200.parallel.dist import DistInfo

CPU = DistInfo(0, 0, 1, torch.device("cpu"), "gloo")


# ----------------------------------------------------------------------------------------------- the flag
def test_the_flag_parses_and_defaults_to_off():
    base = ["--synthetic_data", "4", "--batch_size", "2"]
    assert parse_args(base).activation_checkpointing is False
    assert parse_args(base + ["--activation_checkpointing"]).activation_checkpointing is True
    assert parse_args(base + ["--activation_checkpointing", "true"]).activation_checkpointing is True
    assert parse_args(base + ["--activation_checkpointing", "false"]).activation_checkpointing is False


def test_the_flag_goes_next_to_a_training_config(tmp_path):
    assert "--activation_checkpointing" in ENGINE_FLAGS
    recipe = tmp_path / "recipe.yaml"
    recipe.write_text(yaml.safe_dump(dict(synthetic_data="4", batch_size=2, lr=1e-3)))
    argv = ["--training_config", str(recipe), "--activation_checkpointing", "--engine", "fused"]
    args = parse_args(argv)
    assert args.activation_checkpointing is True and args.batch_size == 2
    with pytest.raises(RuntimeError, match="both a yaml config and command line arguments"):
        parse_args(argv + ["--lr", "1e-2"])  # a training hyper-parameter is still refused next to the recipe


# ----------------------------------------------------------------------------------------------- the module path
def _llama():
    from relora_b200.models import LlamaForCausalLM, SimpleConfig

    return LlamaForCausalLM(SimpleConfig(model_type="llama", vocab_size=96, hidden_size=32, intermediate_size=48,
                                         num_hidden_layers=3, num_attention_heads=2, rms_norm_eps=1e-6, pad_token_id=-1,
                                         max_position_embeddings=32))


def _pythia():
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig

    return GPTNeoXForCausalLM(SimpleConfig(model_type="gpt_neox", vocab_size=96, hidden_size=32, num_hidden_layers=3,
                                           num_attention_heads=2, intermediate_size=128, rotary_pct=0.25, max_position_embeddings=32,
                                           layer_norm_eps=1e-5, use_parallel_residual=True, hidden_act="gelu",
                                           rotary_emb_base=10000, tie_word_embeddings=False))


def _stepper(model, checkpointing: bool):
    from relora_b200.config import build_parser
    from relora_b200.engine.stepper import ModuleStepper, make_stepper

    args = build_parser().parse_args(["--lr", "1e-3", "--gradient_accumulation", "1", "--activation_checkpointing",
                                      str(checkpointing).lower()])
    st = make_stepper(model, CPU, args)
    assert isinstance(st, ModuleStepper)
    return st


@pytest.mark.parametrize("build", [_llama, _pythia], ids=["llama", "pythia"])
def test_module_path_gradients_are_bit_identical_with_checkpointing(build):
    """make_stepper turns on the model's per-layer torch.utils.checkpoint; the recomputed layers redraw the same LoRA-dropout masks
    (the RNG state is restored), so every gradient is the one without checkpointing, bit for bit."""
    from relora_b200.relora import ReLoRaModel

    torch.manual_seed(0)
    model = ReLoRaModel(build(), r=8, lora_alpha=16, lora_dropout=0.1, target_modules=["attn", "attention", "mlp"],
                        init_lora_a="kaiming")
    with torch.no_grad():
        for m in model.relora_modules():
            torch.nn.init.normal_(m.lora_B.weight, std=0.05)
    model.train()
    plain, ckpt = copy.deepcopy(model), model
    st_plain, st_ckpt = _stepper(plain, False), _stepper(ckpt, True)
    inner = ckpt.wrapped_model
    layers = inner.model.layers if hasattr(inner, "model") else inner.gpt_neox.layers
    assert not any(getattr(m, "gradient_checkpointing", False) for m in plain.modules())
    calls = []
    layers[1].register_forward_pre_hook(lambda *_: calls.append(1))
    ids = torch.randint(0, 96, (2, 16), generator=torch.Generator().manual_seed(1))
    torch.manual_seed(5)
    la = st_plain.micro_step(ids)
    torch.manual_seed(5)
    lb = st_ckpt.micro_step(ids)
    assert len(calls) == 2, "the checkpointed layer ran its forward once more in the backward"
    assert torch.equal(la, lb)
    ga = {n: p.grad for n, p in plain.named_parameters() if p.requires_grad}
    gb = {n: p.grad for n, p in ckpt.named_parameters() if p.requires_grad}
    assert set(ga) == set(gb) and any("lora_A" in n for n in ga)
    for n in ga:
        assert ga[n] is not None and torch.equal(ga[n], gb[n]), n


# ----------------------------------------------------------------------------------------------- the fp8 refusal
def test_fp8_frozen_weights_are_refused_with_checkpointing_before_the_device_check():
    from relora_b200.engine import fused_llama
    from relora_b200.relora import ReLoRaModel

    model = ReLoRaModel(_llama(), r=8, lora_alpha=16, lora_dropout=0.1, target_modules=["attn", "mlp"])
    for frozen in ("fp8", "fp8_full"):
        ok, why = fused_llama.supports(model, argparse.Namespace(activation_checkpointing=True, frozen_dtype=frozen))
        assert not ok
        assert why.startswith(f"--activation_checkpointing cannot be combined with --frozen_dtype {frozen}") and "amax" in why
    # each alone gets as far as the shape checks and then the device
    for ns in (argparse.Namespace(activation_checkpointing=True, frozen_dtype=None),
               argparse.Namespace(activation_checkpointing=False, frozen_dtype="fp8")):
        ok, why = fused_llama.supports(model, ns)
        assert not ok and "checkpointing" not in why
