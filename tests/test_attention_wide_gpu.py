"""The wgmma attention kernels at head sizes 72..256 (two to four 64-column panels per head): the head-size refusals, the module
path, the fused executor and the Pythia module path against torch SDPA (run on an H100: -m gpu).  The kernels' numerics at these
head sizes are checked element by element in test_attention_modes_gpu.py."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


@pytest.fixture(scope="module")
def F():
    from relora_b200.ops import fused

    return fused


@pytest.fixture(autouse=True)
def _default_attention_mode(monkeypatch):
    monkeypatch.delenv("RELORA_B200_ATTENTION", raising=False)


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", dtype=torch.float32) * scale).to(BF)


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


@pytest.mark.parametrize("hd", [84, 264])
def test_attention_rejects_unsupported_head_sizes(C, hd):
    B, T, nh = 1, 64, 2
    qkv = torch.zeros(B * T, 3 * nh * hd, device="cuda", dtype=BF)
    out = torch.zeros(B * T, nh * hd, device="cuda", dtype=BF)
    lse = torch.zeros(B, nh, T, device="cuda", dtype=torch.float32)
    with pytest.raises(RuntimeError, match="multiple of 8 and <= 256"):
        C.attention_fwd(qkv, out, lse, B, T, nh, hd, 1.0)
    torch.cuda.synchronize()


@pytest.mark.parametrize("B,nh,T,hd", [(2, 2, 200, 128), (1, 2, 200, 256)])
def test_module_path_attention_at_wide_heads(F, B, nh, T, hd):
    """`F.causal_attention` vs torch SDPA on q, k, v [B, nh, T, hd] incl. the gradients, and the routing of each mode."""
    torch.manual_seed(hd)
    q, k, v = (_rand(B, nh, T, hd).requires_grad_() for _ in range(3))
    assert F.attention_backend(hd, "auto", q) == "sdpa"
    assert F.attention_backend(hd, "native", q) == "native"
    assert F.attention_backend(hd, "sdpa", q) == "sdpa"
    do = _rand(B, nh, T, hd)
    o = F.causal_attention(q, k, v)
    o.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    of = torch.nn.functional.scaled_dot_product_attention(qf, kf, vf, is_causal=True)
    of.backward(do.float())
    assert _relerr(o, of) < 1e-2
    for a, b in ((q.grad, qf.grad), (k.grad, kf.grad), (v.grad, vf.grad)):
        assert _relerr(a, b) < 2e-2


def _llama(hidden, heads, seed=0):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="llama", vocab_size=4096, hidden_size=hidden, intermediate_size=512, num_hidden_layers=2,
                       num_attention_heads=heads, rms_norm_eps=1e-6, pad_token_id=-1, max_position_embeddings=256)
    torch.manual_seed(seed)
    w = ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "mlp"], init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


@pytest.mark.parametrize("hidden,heads", [(640, 8), (256, 2), (512, 2)])
def test_native_attention_matches_sdpa_in_the_executor_at_wide_heads(hidden, heads):
    """head_dim 80, 128, 256: `--attention native` and `sdpa` give the same loss and gradients; `auto` keeps SDPA there."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.ops import fused
    from relora_b200.parallel.dist import DistInfo

    dev = torch.device("cuda", 0)
    info = DistInfo(0, 0, 1, dev, "nccl")
    wa = _llama(hidden, heads)
    wb, wc = copy.deepcopy(wa), copy.deepcopy(wa)
    ids = torch.randint(0, 4096, (3, 128), device=dev)
    fa = FusedLlamaStepper(wa, info, lr=1e-3, grad_accumulation=1, cuda_graphs=True, attention="native")
    fb = FusedLlamaStepper(wb, info, lr=1e-3, grad_accumulation=1, cuda_graphs=False, attention="sdpa")
    fc = FusedLlamaStepper(wc, info, lr=1e-3, grad_accumulation=1, cuda_graphs=False, attention="auto")
    assert fa.native_attn and not fb.native_attn and not fc.native_attn
    fused.seed_state.set(dev, 77)
    la = fa.micro_step(ids)
    fused.seed_state.set(dev, 77)
    lb = fb.micro_step(ids)
    assert abs(float(la) - float(lb)) < 2e-2
    for n, p in zip(fa.trainable_names, fa.trainable_params):
        ga = fa.store.view_like(fa.store.grads, p).float()
        gb = fb.store.view_like(fb.store.grads, fb.trainable_params[fa.trainable_names.index(n)]).float()
        if gb.norm() == 0:
            continue
        assert _relerr(ga, gb) < 0.1, n


def test_pythia_module_path_runs_native_attention_at_head_dim_128(monkeypatch):
    """Tiny GPT-NeoX under ReLoRA (hd 128, partial rotary): RELORA_B200_ATTENTION=native runs the wgmma kernels and matches
    RELORA_B200_ATTENTION=sdpa in loss and LoRA gradients."""
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.ops import fused
    from relora_b200.relora import ReLoRaModel

    torch.manual_seed(0)
    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=2,
                       intermediate_size=1024, rotary_pct=0.25, max_position_embeddings=256, layer_norm_eps=1e-5,
                       use_parallel_residual=True, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=32, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    w = w.to("cuda", BF).train()
    ids = torch.randint(0, 512, (2, 160), device="cuda")
    calls = []
    real = fused.causal_attention
    monkeypatch.setattr(fused, "causal_attention", lambda *a, **k: calls.append(1) or real(*a, **k))
    res = {}
    for mode in ("native", "sdpa"):
        monkeypatch.setenv("RELORA_B200_ATTENTION", mode)
        calls.clear()
        w.zero_grad(set_to_none=True)
        loss = w(input_ids=ids, labels=ids).loss
        loss.backward()
        assert len(calls) == (2 if mode == "native" else 0), (mode, len(calls))
        res[mode] = (float(loss), {n: p.grad.float().clone() for n, p in w.named_parameters() if p.grad is not None and "lora_" in n})
    assert abs(res["native"][0] - res["sdpa"][0]) < 3e-2
    for n, g in res["sdpa"][1].items():
        if g.norm() > 0:
            assert _relerr(res["native"][1][n], g) < 0.08, n
