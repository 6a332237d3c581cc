"""Grouped-query attention on the wgmma kernels (run on an H100: -m gpu): bit-reproducible dK / dV, a column window of a wider
buffer, the interleaved-layout refusal, ``rope_pack_bwd`` with nkv KV heads, and a GQA Llama module path (K/V repeated per query
head) on the native kernels.  Forward and backward over the packed [q: nh | k: nkv | v: nkv] layout are checked element by
element in test_attention_modes_gpu.py."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", dtype=torch.float32) * scale).to(BF)


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


def _run(C, qkv, dout, B, T, nh, nkv, hd):
    """(out, lse, dqkv) of the kernels; every output starts as NaN so an unwritten element shows."""
    scale = 1.0 / math.sqrt(hd)
    out = torch.full((B * T, nh * hd), float("nan"), device="cuda", dtype=BF)
    lse = torch.full((B, nh, T), float("nan"), device="cuda", dtype=torch.float32)
    C.attention_fwd(qkv, out, lse, B, T, nh, hd, scale, nkv=nkv)
    delta = torch.full((B, nh, T), float("nan"), device="cuda", dtype=torch.float32)
    dqkv = torch.full_like(qkv, float("nan"))
    C.attention_bwd(qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, scale, nkv=nkv)
    return out, lse, dqkv


def test_gqa_backward_is_bit_reproducible(C):
    B, T, nh, nkv, hd = 2, 1000, 8, 2, 128
    torch.manual_seed(5)
    qkv = _rand(B * T, (nh + 2 * nkv) * hd)
    dout = _rand(B * T, nh * hd)
    a = _run(C, qkv, dout, B, T, nh, nkv, hd)
    b = _run(C, qkv, dout, B, T, nh, nkv, hd)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_gqa_writes_only_its_window_of_a_wider_buffer(C):
    """qkv / dqkv as column windows of wider NaN-padded buffers: the padding stays NaN, the window matches a dense run."""
    B, T, nh, nkv, hd = 1, 200, 4, 1, 64
    W = (nh + 2 * nkv) * hd
    torch.manual_seed(7)
    dense = _rand(B * T, W)
    dout = _rand(B * T, nh * hd)
    wide = torch.full((B * T, W + 128), float("nan"), device="cuda", dtype=BF)
    wide[:, 64:64 + W].copy_(dense)
    dwide = torch.full_like(wide, float("nan"))
    scale = 1.0 / math.sqrt(hd)
    out = torch.empty(B * T, nh * hd, device="cuda", dtype=BF)
    lse = torch.empty(B, nh, T, device="cuda", dtype=torch.float32)
    C.attention_fwd(wide[:, 64:64 + W], out, lse, B, T, nh, hd, scale, nkv=nkv)
    delta = torch.empty_like(lse)
    C.attention_bwd(wide[:, 64:64 + W], out, dout, lse, delta, dwide[:, 64:64 + W], B, T, nh, hd, scale, nkv=nkv)
    assert dwide[:, :64].isnan().all() and dwide[:, 64 + W:].isnan().all()
    ref = _run(C, dense, dout, B, T, nh, nkv, hd)
    assert torch.equal(out, ref[0]) and torch.equal(dwide[:, 64:64 + W], ref[2])


def test_gqa_refuses_interleaved_layout_and_uneven_groups(C):
    B, T, hd = 1, 64, 64
    out = torch.zeros(B * T, 4 * hd, device="cuda", dtype=BF)
    lse = torch.zeros(B, 4, T, device="cuda", dtype=torch.float32)
    with pytest.raises(RuntimeError, match="interleaved"):
        C.attention_fwd(torch.zeros(B * T, 8 * hd, device="cuda", dtype=BF), out, lse, B, T, 4, hd, 1.0, interleaved=True, nkv=2)
    with pytest.raises(RuntimeError, match="multiple of nkv"):
        C.attention_fwd(torch.zeros(B * T, 10 * hd, device="cuda", dtype=BF), out, lse, B, T, 4, hd, 1.0, nkv=3)
    torch.cuda.synchronize()


@pytest.mark.parametrize("nkv", [1, 2, 4])
def test_rope_pack_bwd_with_kv_heads(C, nkv):
    """dq [B, nh, T, hd], dk / dv [B, nkv, T, hd] -> packed [q | k | v] with the inverse rotation of dq and dk."""
    from relora_b200.models.llama import LlamaRotaryEmbedding, rotate_half

    B, T, nh, hd = 2, 50, 4, 64
    torch.manual_seed(nkv)
    rot = LlamaRotaryEmbedding(hd, 128).to("cuda")
    cos, sin = (t[0, 0].to(BF).contiguous() for t in (rot.cos_cached, rot.sin_cached))
    dq, dk, dv = _rand(B, nh, T, hd), _rand(B, nkv, T, hd), _rand(B, nkv, T, hd)
    out = torch.full((B * T, (nh + 2 * nkv) * hd), float("nan"), device="cuda", dtype=BF)
    C.rope_pack_bwd(dq, dk, dv, out, hd, cos, sin, 0, nkv=nkv)
    c, s = cos[:T].float(), sin[:T].float()
    inv = lambda x: x.float() * c - rotate_half(x.float()) * s  # noqa: E731
    want = torch.cat([inv(dq), inv(dk), dv.float()], dim=1).transpose(1, 2).reshape(B * T, -1)
    assert not out.isnan().any()
    assert (out.float() - want).abs().max() < 3e-2


def test_gqa_llama_module_path_native_matches_sdpa(monkeypatch):
    """A tiny GQA Llama under ReLoRA on the module path (K/V repeated to every query head): RELORA_B200_ATTENTION=native runs
    the wgmma kernels and matches RELORA_B200_ATTENTION=sdpa in loss and gradients."""
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.ops import fused
    from relora_b200.relora import ReLoRaModel

    torch.manual_seed(0)
    cfg = SimpleConfig(model_type="llama", vocab_size=512, hidden_size=512, intermediate_size=768, num_hidden_layers=2,
                       num_attention_heads=8, num_key_value_heads=2, rope_theta=500000.0, max_position_embeddings=256)
    w = ReLoRaModel(LlamaForCausalLM(cfg), r=32, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "mlp"], init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    w = w.to("cuda", BF).train()
    ids = torch.randint(0, 512, (2, 200), device="cuda")
    calls = []
    real = fused.causal_attention
    monkeypatch.setattr(fused, "causal_attention", lambda q, k, v, *a: calls.append(k.shape[1]) or real(q, k, v, *a))
    res = {}
    for mode in ("native", "sdpa"):
        monkeypatch.setenv("RELORA_B200_ATTENTION", mode)
        calls.clear()
        w.zero_grad(set_to_none=True)
        loss = w(input_ids=ids, labels=ids).loss
        loss.backward()
        assert calls == ([8, 8] if mode == "native" else []), (mode, calls)
        res[mode] = (float(loss), {n: p.grad.float().clone() for n, p in w.named_parameters() if p.grad is not None})
    assert abs(res["native"][0] - res["sdpa"][0]) < 3e-2
    for n, g in res["sdpa"][1].items():
        if g.norm() > 0:
            assert _relerr(res["native"][1][n], g) < 0.08, n
