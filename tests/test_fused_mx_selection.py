"""MXFP8-packed frozen weights on the fused Llama executor, the parts that need no GPU: which models `--engine fused --quantize`
takes and the reason for each it refuses, `--engine auto`'s checks left as they were, and the packed stacks' bytes against the
exact quantiser of ops/reference.py."""
import argparse

import pytest
import torch

from relora_b200.engine import fused_llama
from relora_b200.ops import mx
from relora_b200.ops import reference as ref


def _model(quantize="mxfp8", nkv=4, h=256, inter=512, r=128, lora_only=False, trainable_scaling=False, model="llama"):
    from relora_b200.models import GPTNeoXForCausalLM, LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    if model == "llama":
        cfg = SimpleConfig(model_type="llama", vocab_size=512, hidden_size=h, intermediate_size=inter, num_hidden_layers=1,
                           num_attention_heads=4, num_key_value_heads=nkv, rope_theta=10000.0, rms_norm_eps=1e-6, pad_token_id=-1,
                           max_position_embeddings=128)
        base = LlamaForCausalLM(cfg)
    else:
        cfg = SimpleConfig(model_type="gpt_neox", vocab_size=512, hidden_size=h, intermediate_size=4 * h, num_hidden_layers=1,
                           num_attention_heads=4, rotary_pct=0.25, rotary_emb_base=10000, max_position_embeddings=128,
                           layer_norm_eps=1e-5, use_parallel_residual=True, tie_word_embeddings=False)
        base = GPTNeoXForCausalLM(cfg)
    return ReLoRaModel(base, r=r, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "attention", "mlp"],
                       quantize=quantize, lora_only=lora_only, trainable_scaling=trainable_scaling)


def _args(**kw):
    return argparse.Namespace(**{"frozen_dtype": None, "attention": "auto", **kw})


def test_a_quantized_llama_is_taken_up_to_the_device_check():
    """On the CPU every shape check passes and the last check, the device, names the reason."""
    assert fused_llama.supports_quantized(_model(), _args()) == (False, "needs CUDA + bfloat16")
    assert fused_llama.supports_quantized(_model(nkv=2), _args()) == (False, "needs CUDA + bfloat16")  # grouped-query attention
    assert fused_llama.supports_quantized(_model(inter=520), _args()) == (False, "needs CUDA + bfloat16")


@pytest.mark.parametrize("case,kw,args,needle", [
    ("4bit", dict(quantize="4bit"), {}, "only 8bit (mxfp8)"),
    ("nvfp4", dict(quantize="nvfp4"), {}, "4bit (nvfp4) uses --engine module"),
    ("fp8", {}, dict(frozen_dtype="fp8"), "--frozen_dtype fp8 cannot be combined with --quantize"),
    ("fp8_full", {}, dict(frozen_dtype="fp8_full"), "--frozen_dtype fp8_full cannot be combined with --quantize"),
    ("pythia", dict(model="pythia"), {}, "fused for Llama only"),
    ("lora_only", dict(lora_only=True), {}, "lora_only / trainable scaling"),
    ("trainable_scaling", dict(trainable_scaling=True), {}, "lora_only / trainable scaling"),
    ("rank", dict(r=64), {}, "must be multiples of 128 for stacked groups"),
    ("gqa_width", dict(nkv=1, h=256), {}, "grouped-query attention needs num_key_value_heads x head_dim"),
    ("not_quantized", dict(quantize=None), {}, "not quantized"),
    ("intermediate", dict(inter=5461), {}, "intermediate size that is a multiple of 8 (got 5461)"),
])
def test_every_refusal_names_its_reason(case, kw, args, needle):
    ok, why = fused_llama.supports_quantized(_model(**kw), _args(**args))
    assert not ok and needle in why, (case, why)


def test_biased_projections_are_refused():
    m = _model()
    q = m.wrapped_model.model.layers[0].self_attn.q_proj
    q.bias = torch.nn.Parameter(torch.zeros(q.out_features))
    assert fused_llama.supports_quantized(m, _args()) == (False, "biased projections use the module path")


def test_full_rank_is_refused():
    from relora_b200.models import LlamaForCausalLM

    ok, why = fused_llama.supports_quantized(_model().wrapped_model, _args())
    assert not ok and "full-rank training has no frozen weights" in why
    assert isinstance(_model().wrapped_model, LlamaForCausalLM)


def test_auto_keeps_quantized_models_on_the_module_path():
    """`supports()`, the check `--engine auto` consults, still declines every quantised model with its old message."""
    for q in ("8bit", "mxfp8", "4bit"):
        assert fused_llama.supports(_model(quantize=q), _args()) == (
            False, "lora_only / trainable scaling / quantized frozen weights use the module path")


def test_the_constructor_refuses_4bit_and_fp8_with_quantize():
    from relora_b200.engine.fused_llama import FusedLlamaStepper

    with pytest.raises(RuntimeError, match="only mxfp8"):
        FusedLlamaStepper(_model(), None, lr=1e-3, quantize="nvfp4")
    with pytest.raises(RuntimeError, match="cannot be combined with --quantize"):
        FusedLlamaStepper(_model(), None, lr=1e-3, quantize="mxfp8", fp8=True)


# ----------------------------------------------------------------------------------------------- packed stacks
def _parts(shapes, K, seed):
    g = torch.Generator().manual_seed(seed)
    ws = []
    for i, n in enumerate(shapes):
        # a magnitude of its own per 32 x 32 tile, so a scale taken from the wrong tile shows
        e = ((torch.arange(n).unsqueeze(1) // 32 + 3 * (torch.arange(K).unsqueeze(0) // 32) + i) % 7 - 3).float()
        ws.append((torch.randn(n, K, generator=g) * torch.exp2(e)).to(torch.bfloat16))
    return ws


def _packed(w):
    q, f, b = ref.mx_quantize_weight_2d_exact(w)
    return mx.MxWeight(q, f, b, *w.shape)


@pytest.mark.parametrize("shapes,K", [
    ((256, 128, 128), 256),   # q | k | v under grouped-query attention
    ((384, 384, 384), 384),   # q | k | v without it
    ((520, 520), 256),        # gate | up at an intermediate size that is not a multiple of 128
    ((256,), 520),            # down: K not a multiple of 128
])
def test_a_stack_of_packed_modules_is_the_packed_stack(shapes, K):
    """Stacking the modules' packed bytes gives, byte for byte, the quantisation of the stacked matrix (every part on a 128-row
    boundary, zero rows between), including the input-gradient scales, whose blocks interleave the parts'; a part cut back out of
    the stack has the module's own bytes."""
    ws = _parts(shapes, K, len(shapes) * 7 + K)
    parts = [_packed(w) for w in ws]
    st = mx.stack_weights(parts)
    dense = torch.zeros(sum(-(-n // 128) * 128 for n in shapes), K, dtype=torch.bfloat16)
    r0s, r = [], 0
    for w in ws:
        dense[r:r + w.shape[0]] = w
        r0s.append(r)
        r += -(-w.shape[0] // 128) * 128
    q, f, b = ref.mx_quantize_weight_2d_exact(dense)
    assert st.N == dense.shape[0] and st.K == K
    assert torch.equal(st.q, q) and torch.equal(st.sf_fwd, f) and torch.equal(st.sf_bwd, b)
    for p, r0 in zip(parts, r0s):
        cut = mx.stack_part(st, r0, p.N)
        assert cut.q.data_ptr() == st.q[r0].data_ptr()  # an alias, not a copy
        assert torch.equal(cut.q, p.q) and torch.equal(cut.sf_fwd, p.sf_fwd) and torch.equal(cut.sf_bwd, p.sf_bwd)


def test_grouped_lora_segment_of_the_reference_gemm():
    """gemm_mx_ref with n_per_group: output columns of group g take a2's columns g·a2_group_kofs .. + K2."""
    g = torch.Generator().manual_seed(3)
    M, N, K, r = 5, 384, 128, 64
    x = torch.randn(M, K, generator=g).to(torch.bfloat16)
    w = torch.randn(N, K, generator=g).to(torch.bfloat16)
    xq, sfx = ref.mx_quantize_rows_exact(x)
    wq, sfw, _ = ref.mx_quantize_weight_2d_exact(w)
    u = torch.randn(M, 3 * r, generator=g).to(torch.bfloat16)
    B = torch.randn(N, r, generator=g).to(torch.bfloat16)
    got, bound = ref.gemm_mx_ref(xq, sfx, wq, sfw, M, N, K, a2=u, b2=B, n_per_group=128, a2_group_kofs=r)
    base, _ = ref.gemm_mx_ref(xq, sfx, wq, sfw, M, N, K)
    want = base.clone()
    for gi in range(3):
        want[:, gi * 128:(gi + 1) * 128] += u[:, gi * r:(gi + 1) * r].double() @ B[gi * 128:(gi + 1) * 128].double().t()
    assert torch.allclose(got, want, rtol=0, atol=1e-9) and bool((bound >= got.abs() - 1e-9).all())
