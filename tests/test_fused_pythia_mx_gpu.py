"""`--engine fused --quantize 8bit` on the Pythia (GPT-NeoX) executor, on the H100 (-m gpu): the bias epilogue of gemm_mx against
the exact reference, the executor on MXFP8-packed weights against the module path on the same packed bytes and dropout masks,
every MXFP8 call of a micro-step and a merge against the exact contracts, resident memory, and the CLI."""
import copy
import os
import sys

import pytest
import torch

from relora_b200.ops import reference as ref

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_fused_mx_gpu as mxg  # noqa: E402

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
_tiled, _relerr, _gen = mxg._tiled, mxg._relerr, mxg._gen


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


# ----------------------------------------------------------------------------------------------- the bias epilogue of gemm_mx
@pytest.mark.parametrize("M,N,K,mode", [
    (300, 768, 256, "bias"),
    (300, 768, 256, "bias residual"),
    (4100, 768, 384, "bias residual"),      # 33 x 6 tiles: more than the SMs, the persistent loop
    (129, 1024, 256, "bias LoRA"),
    (1000, 768, 512, "bias LoRA residual"),
    (4100, 1536, 256, "bias LoRA grouped"),
    (257, 768, 256, "bias LoRA grouped residual"),
])
def test_gemm_mx_bias_matches_the_exact_reference(C, M, N, K, mode):
    """out = xq·Wᵀ (+ u·Bᵀ, per group) + bias (+ residual), element by element within the fp8 bound."""
    g = _gen(M + N + K)
    r = 128
    grouped = "grouped" in mode
    G = 3 if grouped else 1
    Ng = N // G
    xq, sfx = ref.mx_quantize_rows_exact(_tiled(M, K, g, 1))
    wq, sfw, _ = ref.mx_quantize_weight_2d_exact(_tiled(N, K, g, 32))
    bias = (torch.randn(N, generator=g, device="cuda") * 4).to(BF)
    u = (torch.randn(M, G * r, generator=g, device="cuda") * 0.5).to(BF) if "LoRA" in mode else None
    B = (torch.randn(N, r, generator=g, device="cuda") * 0.1).to(BF) if "LoRA" in mode else None
    res = torch.randn(M, N, generator=g, device="cuda").to(BF) if "residual" in mode else None
    npg, kofs = (Ng, r) if grouped else (0, 0)
    out = torch.full((M, N), float("nan"), dtype=BF, device="cuda")
    C.gemm_mx(xq, sfx, wq, sfw, out, M, N, K, False, u, B, res, npg, kofs, bias)
    want, bound = ref.gemm_mx_ref(xq, sfx, wq, sfw, M, N, K, a2=u, b2=B, residual=res, n_per_group=npg, a2_group_kofs=kofs,
                                  bias=bias)
    ref.assert_gemm_close(out, want, bound, fp8=True)
    # without the bias, the call gives what the form without the argument gives, bit for bit
    a, b = torch.empty_like(out), torch.empty_like(out)
    C.gemm_mx(xq, sfx, wq, sfw, a, M, N, K, False, u, B, res, npg, kofs)
    C.gemm_mx(xq, sfx, wq, sfw, b, M, N, K, False, u, B, res, npg, kofs, None)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_a_bias_with_mn_major_b_is_refused(C):
    M, N, K = 128, 256, 256
    xq = torch.zeros(M, K, dtype=torch.uint8, device="cuda")
    sf = torch.zeros(C.mx_sf_bytes(max(M, N), K), dtype=torch.uint8, device="cuda")
    out = torch.empty(M, N, dtype=BF, device="cuda")
    with pytest.raises(RuntimeError, match="a bias needs K-major B"):
        C.gemm_mx(xq, sf, torch.zeros(K, N, dtype=torch.uint8, device="cuda"), sf, out, M, N, K, True, None, None, None, 0, 0,
                  torch.zeros(N, dtype=BF, device="cuda"))


# ----------------------------------------------------------------------------------------------- the executor
def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _model(p_drop, parallel=True, act="gelu", hidden=256, layers=2, quantize="mxfp8", seed=0):
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=1024, hidden_size=hidden, num_hidden_layers=layers,
                       num_attention_heads=hidden // 64, intermediate_size=4 * hidden, rotary_pct=0.25, max_position_embeddings=64,
                       layer_norm_eps=1e-5, use_parallel_residual=parallel, hidden_act=act, rotary_emb_base=10000,
                       tie_word_embeddings=False)
    torch.manual_seed(seed)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=p_drop, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming", quantize=quantize)
    with torch.no_grad():
        for mod in w.relora_modules():
            torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
            torch.nn.init.normal_(mod.bias, std=0.02)
        for n, p in w.named_parameters():
            if "layernorm" in n or "layer_norm" in n:
                p.add_(torch.randn_like(p) * 0.05)
    return w.cuda().to(BF).train()


def _grads(st):
    return {n: st.store.view_like(st.store.grads, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


def _params(st, flat):
    return {n: st.store.view_like(flat, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


@pytest.mark.parametrize("parallel,p_drop,graphs,T,act", [
    (True, 0.0, False, 96, "gelu"),
    (True, 0.1, True, 96, "gelu"),
    (False, 0.1, False, 80, "gelu_new"),
    (False, 0.0, True, 96, "gelu"),
    (True, 0.1, False, 80, "gelu_new"),
])
def test_fused_mx_pythia_matches_the_module_path(parallel, p_drop, graphs, T, act):
    """Fused-MX against ModuleStepper on the same packed bytes and dropout masks (parallel and sequential residual, erf and tanh
    GELU, a ragged T beyond max_position_embeddings), then an update, a second step and evaluation."""
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused, mx

    dev = torch.device("cuda", 0)
    wa = _model(p_drop, parallel, act)
    wb = copy.deepcopy(wa)
    fs = FusedPythiaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs, quantize="mxfp8")
    ms = ModuleStepper(wb, _info(), lr=1e-3, grad_accumulation=1, native=fused.NativeOptim())
    for ma, mb in zip(wa.relora_modules(), wb.relora_modules()):  # the executor runs on the module path's bytes
        assert isinstance(ma.qweight, mx.MxWeight)
        assert torch.equal(ma.qweight.q, mb.qweight.q) and torch.equal(ma.qweight.sf_fwd, mb.qweight.sf_fwd)
        assert torch.equal(ma.qweight.sf_bwd, mb.qweight.sf_bwd)
    ids = torch.randint(0, 1024, (2, T), generator=torch.Generator().manual_seed(T)).to(dev)
    fused.seed_state.set(dev, 4321)
    la = fs.micro_step(ids)
    fused.seed_state.set(dev, 4321)
    lb = ms.micro_step(ids)
    assert abs(float(la) - float(lb)) < 4e-2, (float(la), float(lb))
    ga, gb = _grads(fs), _grads(ms)
    assert set(ga) == set(gb)
    errs = {n: _relerr(ga[n], gb[n]) for n in ga if gb[n].norm() > 0}
    assert max(errs.values()) < 0.15, sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    for key in ("query_key_value.bias", "dense_4h_to_h.bias", "input_layernorm.bias", "lora_A", "embed_in.weight"):
        assert any(key in n and gb[n].norm() > 0 for n in gb), key
    before = fs.store.params.clone()
    fs.update()
    ms.update()
    assert not torch.equal(before, fs.store.params)
    pa, pb, p0 = _params(fs, fs.store.params), _params(ms, ms.store.params), _params(fs, before)
    nh = wa.wrapped_model.config.num_attention_heads
    cos = {}
    for n in pa:  # AdamW's first step moves each entry by about lr·sign(g): the steps are compared by direction
        da, db = (pa[n] - p0[n]).flatten(), (pb[n] - p0[n]).flatten()
        if n.endswith("query_key_value.bias"):
            # the key bias adds the same q·b_k to every logit of a query, so softmax removes it: its exact gradient is zero and
            # the step either path takes is the sign of rounding noise; the q and v thirds are compared
            qv = torch.ones(nh, 3, da.numel() // (3 * nh), dtype=torch.bool, device=da.device)
            qv[:, 1] = False
            da, db = da[qv.flatten()], db[qv.flatten()]
        if db.norm() > 0:
            cos[n] = float(torch.dot(da, db) / (da.norm() * db.norm()))
    assert min(cos.values()) > 0.9, sorted(cos.items(), key=lambda kv: kv[1])[:5]
    fused.seed_state.set(dev, 99)
    l2 = fs.micro_step(ids)  # graph replay when graphs are on
    fused.seed_state.set(dev, 99)
    l2m = ms.micro_step(ids)
    assert torch.isfinite(l2) and abs(float(l2) - float(l2m)) < 4e-2, (float(l2), float(l2m))
    ev, evm = fs.eval_loss(ids), ms.eval_loss(ids)
    assert torch.isfinite(ev) and abs(float(ev) - float(evm)) < 4e-2, (float(ev), float(evm))


class _Audit(mxg._Audit):
    """The Llama audit with gemm_mx's trailing bias operand."""

    def _gemm_mx(self, b, a):
        xa, sfa, wb, sfb, _, M, N, K, mn = b[:9]
        a2, b2, res = (list(b[9:12]) + [None] * 3)[:3]
        npg, kofs, bias = (list(b[12:15]) + [0, 0, None])[:3]
        want, bound = ref.gemm_mx_ref(xa, sfa, wb, sfb, M, N, K, mn, a2, b2, res, n_per_group=npg, a2_group_kofs=kofs, bias=bias)
        ref.assert_gemm_close(a[4][:M, :N], want, bound, fp8=True)
        return f"gemm_mx {'MN' if mn else 'K'}-major{' LoRA' if a2 is not None else ''}{' grouped' if npg else ''}" \
               f"{' bias' if bias is not None else ''}{' residual' if res is not None else ''}"


@pytest.mark.parametrize("parallel", [True, False])
def test_every_mx_call_of_a_micro_step_and_a_merge_matches_the_contract(C, monkeypatch, parallel):
    """One fused micro-step with dropout and one merge: every MXFP8 call checked.  mx_quantize_rows runs once for each of the
    four projection inputs and each of the four output gradients; each merge's bytes, which the module's packed weight is, are the
    exact requantisation of the old bytes plus the executor's delta, and that delta is s·B·A."""
    from relora_b200.engine.fused_pythia import FusedPythiaStepper
    from relora_b200.ops import fused

    w = _model(0.1, parallel)
    fs = FusedPythiaStepper(w, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False, quantize="mxfp8")
    mods = list(w.relora_modules())
    old = [(m.qweight.q.clone(), m.qweight.sf_fwd.clone()) for m in mods]
    AB = [(m.lora_A.weight.detach().float().clone(), m.lora_B.weight.detach().float().clone()) for m in mods]
    audit = _Audit(C, monkeypatch)
    fused.seed_state.set(torch.device("cuda", 0), 77)
    fs.micro_step(torch.randint(0, 1024, (2, 96), generator=torch.Generator().manual_seed(3)).cuda())
    fs.merge_and_reinit()
    torch.cuda.synchronize()
    print(f"[fused pythia mx audit] {dict(sorted(audit.modes.items()))}")
    L = len(fs.layers)
    assert audit.modes["merge"] == 4 * L
    assert audit.modes["quantize_rows"] == 8 * L
    assert audit.modes["gemm_mx K-major LoRA bias"] == 2 * L            # query_key_value, dense_h_to_4h
    assert audit.modes["gemm_mx K-major LoRA bias residual"] == 2 * L   # dense, dense_4h_to_h
    assert audit.modes["gemm_mx MN-major"] == 4 * L                     # the input gradients
    s = fs.scale
    for l, S in enumerate(fs.layers):
        for i, m in enumerate(S.mods):
            j = mods.index(m)
            d = audit.deltas[4 * l + i]
            A, B = AB[j]
            assert _relerr(d, s * (B @ A)) < 1e-5
            q, f, bw = ref.mx_quantize_weight_2d_exact(q_old=old[j][0], sf_old=old[j][1], delta=d, N=m.out_features, K=m.in_features)
            ref.assert_e4m3_bytes_equal("module q", m.qweight.q[:q.shape[0], :q.shape[1]], q)
            ref.assert_bitwise_equal("module sf_fwd", m.qweight.sf_fwd, f)
            ref.assert_bitwise_equal("module sf_bwd", m.qweight.sf_bwd, bw)
            assert m.qweight is fs.Wmx[l][i] and m.qweight.q.data_ptr() == getattr(S, "W_" + ("qkv", "o", "h", "4")[i]).q.data_ptr()
            assert float(m.lora_B.weight.float().abs().max()) == 0.0


def test_packed_weights_are_the_only_resident_frozen_weights():
    """No bf16 frozen weight exists, and the device memory after construction is below the bf16 executor's on the same model by
    at least 90 % of the bytes packing saves."""
    import gc

    from relora_b200.engine.fused_pythia import FusedPythiaStepper

    def build(quantize):
        gc.collect()
        torch.cuda.empty_cache()
        m = _model(0.0, hidden=512, layers=4, quantize=quantize)
        fs = FusedPythiaStepper(m, _info(), lr=1e-3, cuda_graphs=False, quantize=quantize)
        torch.cuda.synchronize()
        return m, fs, torch.cuda.memory_allocated()

    m, fs, bf16_alloc = build(None)
    frozen_bf16 = sum(mod.weight.numel() * 2 for mod in m.relora_modules())
    del m, fs
    m, fs, mx_alloc = build("mxfp8")
    packed = sum(mod.qweight.nbytes for mod in m.relora_modules())
    for mod in m.relora_modules():
        assert "weight" not in mod._parameters and mod.qweight.q.dtype == torch.uint8
    for S in fs.layers:
        assert all(getattr(S, "W_" + t).q.dtype == torch.uint8 for t in ("qkv", "o", "h", "4"))
    saved = bf16_alloc - mx_alloc
    print(f"[fused pythia mx memory] bf16 executor {bf16_alloc / 2**20:.1f} MiB, mx {mx_alloc / 2**20:.1f} MiB, "
          f"frozen bf16 {frozen_bf16 / 2**20:.1f} MiB, packed {packed / 2**20:.1f} MiB")
    assert saved >= 0.9 * (frozen_bf16 - packed), (saved, frozen_bf16, packed)


# ----------------------------------------------------------------------------------------------- command line
def test_cli_pythia_recipe_with_8bit_weights_on_the_fused_executor(tmp_path):
    """The toy form of the shipped recipe (Pythia warm start, Megatron data, magnitude pruning, autoresume) with quantize: 8bit
    and --engine fused: two restarts, dense bf16 checkpoint weights, and a resumed run."""
    import yaml

    from test_neox_data import _tiny_pythia_dir, _write_corpus
    from torchrun_main import main

    ckpt = _tiny_pythia_dir(str(tmp_path / "pythia-tiny"), hidden=128, heads=2)
    prefix = str(tmp_path / "pile")
    _write_corpus(prefix, n_docs=400, vocab=512, seed=11)
    data = tmp_path / "data.yaml"
    data.write_text(yaml.safe_dump({"data-path": prefix, "split": "8,1,1", "data-impl": "mmap", "seq-length": 64, "train-iters": 20,
                                    "eval-interval": 5, "eval-iters": 1}))
    recipe = tmp_path / "recipe.yaml"
    recipe.write_text(yaml.safe_dump(dict(
        model_name_or_path=ckpt, model_revision="step1000", dtype="bfloat16", distributed_type="ddp",
        megatron_dataset_config=str(data), max_length=64, workers=0, quantize="8bit",
        use_peft=True, lora_r=128, relora=3, force_keep_original=True, restart_warmup_steps=1, reset_optimizer_on_relora=False,
        optimizer_magnitude_pruning=0.8, optimizer="adam", lr=4e-4, adam_beta1=0.9, adam_beta2=0.95, weight_decay=0.01,
        scheduler="cosine_restarts", warmup_steps=2, batch_size=2, total_batch_size=4, num_training_steps=9,
        save_dir=str(tmp_path / "run"), autoresume=True, save_every=3, eval_every=3, tags="relora1b", comment="toy")))
    res = main(["--training_config", str(recipe), "--device", "cuda", "--engine", "fused"])
    assert res["executor"] == "FusedPythiaStepper" and res["update_step"] == 9 and res["n_lora_restarts"] == 2
    assert res["final_eval_loss"] < 7.5  # ln(512) = 6.24 at init
    sd = torch.load(os.path.join(str(tmp_path / "run"), "model_9", "pytorch_model.bin"), weights_only=True)
    keys = [f"gpt_neox.layers.{l}.{m}.weight" for l in range(2)
            for m in ("attention.query_key_value", "attention.dense", "mlp.dense_h_to_4h", "mlp.dense_4h_to_h")]
    for k in keys:
        w = sd[k]
        assert w.dim() == 2 and w.dtype == BF and bool(torch.isfinite(w.float()).all()), k
    assert sd["gpt_neox.layers.0.attention.query_key_value.weight"].shape == (384, 128)
    recipe.write_text(recipe.read_text().replace("num_training_steps: 9", "num_training_steps: 12"))
    res2 = main(["--training_config", str(recipe), "--device", "cuda", "--engine", "fused"])
    assert res2["executor"] == "FusedPythiaStepper" and res2["update_step"] == 12
    assert "model_12" in os.listdir(str(tmp_path / "run"))
