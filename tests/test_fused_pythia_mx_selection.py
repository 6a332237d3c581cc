"""MXFP8-packed frozen weights on the fused Pythia (GPT-NeoX) executor, the parts that need no GPU: which models
`--engine fused --quantize` takes and the reason for each it refuses, the Llama executor's checks and `--engine auto`'s left as they
were, and the constructor's refusals."""
import argparse

import pytest
import torch

from relora_b200.engine import fused_llama, fused_pythia


def _model(quantize="mxfp8", h=256, inter=None, r=128, lora_only=False, trainable_scaling=False, parallel=True, act="gelu",
           hidden_dropout=0.0, rotary_pct=0.25, heads=4, model="pythia"):
    from relora_b200.models import GPTNeoXForCausalLM, LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    if model == "llama":
        cfg = SimpleConfig(model_type="llama", vocab_size=512, hidden_size=h, intermediate_size=inter or 512, num_hidden_layers=1,
                           num_attention_heads=4, num_key_value_heads=4, rope_theta=10000.0, rms_norm_eps=1e-6, pad_token_id=-1,
                           max_position_embeddings=128)
        base = LlamaForCausalLM(cfg)
    else:
        cfg = SimpleConfig(model_type="gpt_neox", vocab_size=512, hidden_size=h, intermediate_size=inter or 4 * h, num_hidden_layers=1,
                           num_attention_heads=heads, rotary_pct=rotary_pct, rotary_emb_base=10000, max_position_embeddings=128,
                           layer_norm_eps=1e-5, use_parallel_residual=parallel, tie_word_embeddings=False, hidden_act=act,
                           hidden_dropout=hidden_dropout, attention_dropout=0.0)
        base = GPTNeoXForCausalLM(cfg)
    return ReLoRaModel(base, r=r, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "attention", "mlp"],
                       quantize=quantize, lora_only=lora_only, trainable_scaling=trainable_scaling)


def _args(**kw):
    return argparse.Namespace(**{"frozen_dtype": None, "attention": "auto", **kw})


@pytest.mark.parametrize("kw", [{}, dict(parallel=False), dict(quantize="8bit"), dict(act="gelu_new")])
def test_a_quantized_pythia_is_taken_up_to_the_device_check(kw):
    """On the CPU every other check passes (parallel and sequential residual, both spellings of the 8-bit format, tanh GELU) and
    the last check, the device, names the reason."""
    assert fused_pythia.supports_quantized(_model(**kw), _args()) == (False, "needs CUDA + bfloat16")


@pytest.mark.parametrize("case,kw,args,needle", [
    ("4bit", dict(quantize="4bit"), {}, "only 8bit (mxfp8)"),
    ("nvfp4", dict(quantize="nvfp4"), {}, "4bit (nvfp4) uses --engine module"),
    ("fp8", {}, dict(frozen_dtype="fp8"), "--frozen_dtype fp8 cannot be combined with --quantize"),
    ("fp8_full", {}, dict(frozen_dtype="fp8_full"), "--frozen_dtype fp8_full cannot be combined with --quantize"),
    ("not_quantized", dict(quantize=None), {}, "not quantized"),
    ("lora_only", dict(lora_only=True), {}, "lora_only / trainable scaling"),
    ("trainable_scaling", dict(trainable_scaling=True), {}, "lora_only / trainable scaling"),
    ("llama", dict(model="llama"), {}, "not a GPT-NeoX (Pythia) model"),
    ("dropout", dict(hidden_dropout=0.1), {}, "hidden / attention dropout must be 0"),
    ("activation", dict(act="relu"), {}, "only the GELU activation is fused"),
    ("rank", dict(r=64), {}, "rank (64) must be multiples of 128"),
    ("intermediate", dict(inter=1000), {}, "intermediate (1000)"),
    ("hidden_128", dict(h=192, heads=4), {}, "hidden (192)"),
    ("hidden_2048", dict(h=2176, heads=17), {}, "must be <= 2048 (LayerNorm kernel limit)"),
    ("head_dim", dict(h=256, heads=64), {}, "head_dim (4) must be a multiple of 8"),
    ("rotary", dict(rotary_pct=0.3), {}, "rotary dims must be even"),
])
def test_every_refusal_names_its_reason(case, kw, args, needle):
    ok, why = fused_pythia.supports_quantized(_model(**kw), _args(**args))
    assert not ok and needle in why, (case, why)


def test_full_rank_is_refused():
    ok, why = fused_pythia.supports_quantized(_model().wrapped_model, _args())
    assert not ok and "full-rank training has no frozen weights" in why


def test_bias_less_projections_are_refused():
    m = _model()
    m.wrapped_model.gpt_neox.layers[0].attention.dense.bias = None
    assert fused_pythia.supports_quantized(m, _args()) == (False, "projections without bias use the module path")


def test_the_other_checks_are_unchanged_for_quantized_models():
    """The Llama executor still names Pythia as the model it does not take, and `supports()` (what `--engine auto` consults)
    still declines every quantised Pythia with its old message."""
    for q in ("8bit", "mxfp8", "4bit"):
        ok, why = fused_llama.supports_quantized(_model(quantize=q), _args())
        assert not ok and "fused for Llama only" in why
        assert fused_pythia.supports(_model(quantize=q), _args()) == (
            False, "lora_only / trainable scaling / quantized frozen weights use the module path")


def test_the_constructor_refuses_4bit_and_fp8_with_quantize():
    from relora_b200.engine.fused_pythia import FusedPythiaStepper

    with pytest.raises(RuntimeError, match="only mxfp8"):
        FusedPythiaStepper(_model(), None, lr=1e-3, quantize="nvfp4")
    with pytest.raises(RuntimeError, match="cannot be combined with --quantize"):
        FusedPythiaStepper(_model(), None, lr=1e-3, quantize="mxfp8", fp8=True)
    with pytest.raises(RuntimeError, match="needs CUDA"):  # a valid request on the CPU stops at the device
        FusedPythiaStepper(_model(), None, lr=1e-3, quantize="mxfp8")


def test_the_reference_gemm_adds_the_bias_before_the_residual():
    """gemm_mx_ref with a bias: out[m, n] gains bias[n] and the bound |bias[n]|; without it the result is what it was."""
    from relora_b200.ops import reference as ref

    g = torch.Generator().manual_seed(11)
    M, N, K = 7, 256, 128
    xq, sfx = ref.mx_quantize_rows_exact(torch.randn(M, K, generator=g).to(torch.bfloat16))
    wq, sfw, _ = ref.mx_quantize_weight_2d_exact(torch.randn(N, K, generator=g).to(torch.bfloat16))
    bias = torch.randn(N, generator=g).to(torch.bfloat16)
    res = torch.randn(M, N, generator=g).to(torch.bfloat16)
    base, bb = ref.gemm_mx_ref(xq, sfx, wq, sfw, M, N, K, residual=res)
    got, gb = ref.gemm_mx_ref(xq, sfx, wq, sfw, M, N, K, residual=res, bias=bias)
    assert torch.equal(got, base + bias.double()) and torch.equal(gb, bb + bias.double().abs())
