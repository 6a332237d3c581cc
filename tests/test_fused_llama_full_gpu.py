"""Full-rank training on the fused Llama executor (H100: -m gpu): selection, gradients and updates against the module path, the
zero padding of the MLP blocks, determinism, every GEMM call against the reference, and a warm-up followed by ReLoRA through the
command line."""
import copy
import json
import os

import pytest
import torch

from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
VOCAB = 4096


def _relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def _cfg(inter=512, nkv=4, hidden=256, nh=4, layers=2):
    from relora_b200.models import SimpleConfig

    return SimpleConfig(model_type="llama", vocab_size=VOCAB, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
                        num_attention_heads=nh, num_key_value_heads=nkv, rms_norm_eps=1e-6, pad_token_id=-1, max_position_embeddings=256)


def _llama(inter=512, nkv=4, seed=0):
    from relora_b200.models import LlamaForCausalLM

    torch.manual_seed(seed)
    return LlamaForCausalLM(_cfg(inter, nkv)).cuda().to(BF)


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _fused(model, **kw):
    from relora_b200.engine.fused_llama import FusedLlamaStepper

    kw.setdefault("lr", 1e-3)
    kw.setdefault("grad_accumulation", 1)
    return FusedLlamaStepper(model, _info(), **kw)


def _module(model, **kw):
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    kw.setdefault("lr", 1e-3)
    kw.setdefault("grad_accumulation", 1)
    return ModuleStepper(model, _info(), native=fused.NativeOptim() if next(model.parameters()).dtype == BF else None, **kw)


def _grads(st):
    return {n: st.store.view_like(st.store.grads, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


def _padding(st, p, flat):
    """The zero-padded part of parameter ``p``'s storage block in ``flat`` (params or grads of the store)."""
    o, n = st.store.segment(p)
    rs, cs = st.store.storage[id(p)]
    block = flat[o:o + n].view(rs, cs)
    return torch.cat([block[p.shape[0]:].flatten(), block[:, p.shape[1]:].flatten()])


def test_selection():
    """`auto` keeps full-rank Llama on the module path; `fused` builds the full-rank executor."""
    from argparse import Namespace

    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper, make_stepper

    def args(engine):
        return Namespace(engine=engine, optimizer="adam", comm="auto", lr=1e-3, adam_beta1=0.9, adam_beta2=0.999, weight_decay=0.0,
                         clip_grad_norm=1.0, gradient_accumulation=1, cuda_graphs=False, attention="auto", frozen_dtype=None,
                         deterministic=False)

    assert type(make_stepper(_llama(), _info(), args("auto"))) is ModuleStepper
    st = make_stepper(_llama(), _info(), args("fused"))
    assert type(st) is FusedLlamaStepper and st.full
    with pytest.raises(RuntimeError, match="frozen weights"):
        make_stepper(_llama(), _info(), Namespace(**{**vars(args("fused")), "frozen_dtype": "fp8"}))


def test_stacked_views_alias_the_module_parameters():
    """Wqkv covers unequal q / k / v blocks (GQA), Wgu / Wd the zero-padded gate / up / down blocks (341 -> 384)."""
    m = _llama(inter=341, nkv=1)
    st = _fused(m, cuda_graphs=False)
    h, kv, fp = 256, 64, 384
    for layer, S in zip(m.model.layers, st.layers):
        at, mlp = layer.self_attn, layer.mlp
        assert S.Wqkv.shape == (h + 2 * kv, h) and S.gWqkv.shape == S.Wqkv.shape and S.gWqkv.dtype == torch.float32
        for w, r0 in ((at.q_proj.weight, 0), (at.k_proj.weight, h), (at.v_proj.weight, h + kv)):
            assert w.data_ptr() == S.Wqkv[r0:].data_ptr() and w.stride() == (h, 1)
        assert at.o_proj.weight.data_ptr() == S.Wo.data_ptr()
        assert S.Wgu.shape == (2 * fp, h) and mlp.gate_proj.weight.data_ptr() == S.Wgu.data_ptr()
        assert mlp.up_proj.weight.data_ptr() == S.Wgu[fp:].data_ptr() and mlp.up_proj.weight.shape == (341, h)
        assert S.Wd.shape == (h, fp) and mlp.down_proj.weight.data_ptr() == S.Wd.data_ptr() and mlp.down_proj.weight.stride() == (fp, 1)
        assert float(S.Wgu[341:fp].abs().sum()) == 0 and float(S.Wd[:, 341:].abs().sum()) == 0
        for p in (mlp.gate_proj.weight, mlp.up_proj.weight, mlp.down_proj.weight):
            assert st.store.is_padded(p)
    assert st.lora_params == [] and st.Wqkv is None
    with pytest.raises(RuntimeError, match="ReLoRA"):
        st.merge_and_reinit()


@pytest.mark.parametrize("attention", ["native", "sdpa"])
@pytest.mark.parametrize("graphs", [False, True])
@pytest.mark.parametrize("nkv", [4, 1])
@pytest.mark.parametrize("inter", [512, 341])
def test_gradients_match_the_fp32_module_path(inter, nkv, graphs, attention):
    """One micro-step on identical weights.  Reference: the same model in fp32 on the module path.  Each fused gradient (and the
    loss) may be off by at most twice the bf16 module path's own error, with a floor of 1e-2."""
    mb = _llama(inter, nkv)
    mf, m32 = copy.deepcopy(mb), copy.deepcopy(mb).float()
    ids = torch.randint(0, VOCAB, (3, 128), device="cuda")
    l32 = m32(input_ids=ids, labels=ids).loss
    l32.backward()
    g32 = {n: p.grad for n, p in m32.named_parameters()}
    ms = _module(mb)
    lb = ms.micro_step(ids)
    st = _fused(mf, cuda_graphs=graphs, attention=attention)
    assert st.native_attn == (attention == "native")
    lf = st.micro_step(ids)
    e_mod, e_fus = abs(float(lb) - float(l32)) / float(l32), abs(float(lf) - float(l32)) / float(l32)
    assert e_fus <= max(2 * e_mod, 1e-2), ("loss", e_fus, e_mod)
    gb, gf = _grads(ms), _grads(st)
    assert set(gf) == set(g32)
    worst = 0.0
    for n in g32:
        e_mod, e_fus = _relerr(gb[n], g32[n]), _relerr(gf[n], g32[n])
        worst = max(worst, e_fus)
        assert e_fus <= max(2 * e_mod, 1e-2), (n, e_fus, e_mod)
    print(f"[full rank] inter={inter} nkv={nkv} graphs={graphs} {attention}: worst gradient relative error {worst:.3g}")
    for layer in mf.model.layers if inter == 341 else ():
        for p in (layer.mlp.gate_proj.weight, layer.mlp.up_proj.weight, layer.mlp.down_proj.weight):
            assert float(_padding(st, p, st.store.grads).abs().sum()) == 0


def test_updates_track_the_module_path_and_keep_the_padding_zero(tmp_path):
    """5 updates with gradient accumulation 2 (weight decay on, graphs on).  Each parameter's distance from an fp32 module-path run
    may be at most twice the bf16 module path's distance, with a floor of 1e-2; the padded rows / columns of gate / up / down stay
    exactly zero; the module parameters (strided views of the store) save and load in the reference layout."""
    from relora_b200.models import LlamaForCausalLM

    mb = _llama(inter=341, nkv=1)
    mf, m32 = copy.deepcopy(mb), copy.deepcopy(mb).float()
    kw = dict(lr=1e-3, weight_decay=0.1, grad_accumulation=2)
    steppers = {"fp32": _module(m32, **kw), "module": _module(mb, **kw), "fused": _fused(mf, cuda_graphs=True, **kw)}
    g = torch.Generator(device="cuda").manual_seed(5)
    batches = [torch.randint(0, VOCAB, (2, 96), device="cuda", generator=g) for _ in range(10)]
    for i, ids in enumerate(batches):
        for st in steppers.values():
            st.micro_step(ids)
            if i % 2 == 1:
                st.update()
    p32 = dict(m32.named_parameters())
    worst = 0.0
    for (n, pm), pf in zip(mb.named_parameters(), mf.parameters()):
        d_mod, d_fus = _relerr(pm, p32[n]), _relerr(pf, p32[n])
        worst = max(worst, d_fus)
        assert d_fus <= max(2 * d_mod, 1e-2), (n, d_fus, d_mod)
    print(f"[full rank] after 5 updates: worst parameter relative distance from fp32 {worst:.3g}")
    st = steppers["fused"]
    for layer in mf.model.layers:
        for p in (layer.mlp.gate_proj.weight, layer.mlp.up_proj.weight, layer.mlp.down_proj.weight):
            for flat in (st.store.params, st.optimizer.exp_avg, st.optimizer.exp_avg_sq):
                pad = _padding(st, p, flat)
                assert pad.numel() > 0 and torch.equal(pad, torch.zeros_like(pad))
    before = {k: v.clone() for k, v in mf.state_dict().items()}
    mf.save_pretrained(str(tmp_path / "m"))
    back = LlamaForCausalLM.from_pretrained(str(tmp_path / "m"))
    for k, v in back.state_dict().items():
        assert torch.equal(v.cpu(), before[k].cpu()), k
    assert back.model.layers[0].mlp.down_proj.weight.shape == (256, 341)


def test_deterministic_mode_is_bit_reproducible():
    """`deterministic=True` (no split-K in the weight gradients): two runs from the same seed give bit-identical gradients and,
    after an update without clipping, bit-identical parameters.  The [h]-sized RMSNorm weight gradients are combined with
    vector atomics and are excluded, like in the ReLoRA test of this mode; the same holds for parameters after more than one
    update, since the norm weights feed every later step."""
    ids = torch.randint(0, VOCAB, (3, 128), device="cuda")
    runs = []
    for _ in range(2):
        m = _llama(inter=341, nkv=1, seed=3)
        st = _fused(m, cuda_graphs=True, deterministic=True, clip_grad_norm=0.0)
        assert st.wgrad_split_k == 1
        st.micro_step(ids)
        torch.cuda.synchronize()
        g = {n: v.clone() for n, v in _grads(st).items()}
        st.update()
        torch.cuda.synchronize()
        runs.append((g, {n: p.detach().clone() for n, p in m.named_parameters()}))
    for n in runs[0][0]:
        if n.endswith("norm.weight"):
            continue
        assert torch.equal(runs[0][0][n], runs[1][0][n]), n
        assert torch.equal(runs[0][1][n], runs[1][1][n]), n


# the GEMM modes of one full-rank micro-step and evaluation: projections with the residual epilogue, input gradients reading W
# MN-major, fp32 weight gradients accumulated from two MN-major operands (split-K unless deterministic); no K2 (LoRA) segment,
# no per-group windows, no bias, no fp8
_FULL_MODES = {"residual", "b1_mn", "a1_mn", "accumulate", "split_k"}


@pytest.mark.parametrize("deterministic", [False, True])
def test_every_gemm_call_matches_the_reference(deterministic, monkeypatch):
    """Every gemm call of one full-rank micro-step and one evaluation (GQA, padded MLP), replayed on clones of its inputs against
    ops.reference.gemm_ref; the set of modes is the expected one, and no LoRA input-gradient kernel runs."""
    from relora_b200.ops import fused

    C = fused._C()
    st = _fused(_llama(inter=341, nkv=1), cuda_graphs=False, deterministic=deterministic)
    gemm0 = fused.gemm
    seen = {"calls": 0, "worst": 0.0, "modes": set()}

    def audited(a1, b1, out=None, **kw):
        torch.cuda.synchronize()  # the weight gradients run on the side stream
        cl = lambda v: v.clone() if torch.is_tensor(v) else v  # noqa: E731
        a1c, b1c, kwc, prev = cl(a1), cl(b1), {k: cl(v) for k, v in kw.items()}, cl(out)
        res = gemm0(a1, b1, out, **kw)
        torch.cuda.synchronize()
        want, bound = ref.gemm_ref(a1c, b1c, prev, **kwc)
        seen["worst"] = max(seen["worst"], ref.assert_gemm_close(res, want, bound))
        seen["calls"] += 1
        for k, v in kw.items():
            if k == "split_k":
                if v != 1:
                    seen["modes"].add(k)
            elif k not in ("M", "N", "K1") and v is not None and v is not False and not (type(v) in (int, float) and v == 0):
                seen["modes"].add(k)
        return res

    def no_lora_dx(*a, **k):
        raise AssertionError("full-rank training has no LoRA input gradient")

    monkeypatch.setattr(fused, "gemm", audited)
    monkeypatch.setattr(C, "lora_dx", no_lora_dx)
    ids = torch.randint(0, VOCAB, (3, 97), device="cuda")
    loss = st.micro_step(ids)
    n_train = seen["calls"]
    ev = st.eval_loss(ids)
    assert torch.isfinite(loss) and torch.isfinite(ev)
    print(f"[gemm modes] full rank deterministic={deterministic}: {seen['calls']} calls, worst ratio {seen['worst']:.3g}, "
          f"modes {sorted(seen['modes'])}")
    assert seen["modes"] == (_FULL_MODES - {"split_k"} if deterministic else _FULL_MODES)
    # per layer: 4 projections, 4 input gradients, 4 weight gradients (qkv one launch under GQA); LM head: 3 per 4096-token chunk
    assert n_train == 2 * 12 + 3 and seen["calls"] - n_train == 2 * 4 + 1


def test_warmup_then_relora_through_the_command_line(tmp_path):
    """A tiny Llama trains full-rank on the fused executor (adam_zero, --deterministic, SDPA) and saves; ReLoRA continues from it
    as --warmed_up_model on the fused executor; the warm-up checkpoint loads strictly into a module-path model bit for bit;
    --autoresume (skipping one batch) continues the warm-up.  Two KV heads: the ReLoRA executor needs nkv·head_dim to be a
    multiple of 128."""
    from relora_b200 import ckpt as ckpt_lib
    from relora_b200.models import LlamaForCausalLM, load_config
    from relora_b200.models.llama import load_state_dict_files
    from torchrun_main import main

    cfg = tmp_path / "tiny.json"
    cfg.write_text(json.dumps(dict(architectures=["LlamaForCausalLM"], model_type="llama", hidden_size=256, intermediate_size=341,
                                   num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2, rms_norm_eps=1e-6,
                                   vocab_size=VOCAB, pad_token_id=-1, max_position_embeddings=256, initializer_range=0.02)))
    warm, rel = str(tmp_path / "warm"), str(tmp_path / "relora")
    common = ["--model_config", str(cfg), "--synthetic_data", str(VOCAB), "--batch_size", "4", "--total_batch_size", "8",
              "--max_length", "128", "--lr", "1e-3", "--scheduler", "cosine", "--warmup_steps", "2", "--eval_every", "100",
              "--dtype", "bfloat16", "--workers", "0", "--engine", "fused"]

    def warmup(steps, *extra):
        return main(common + ["--num_training_steps", str(steps), "--save_every", "4", "--save_dir", warm, "--optimizer", "adam_zero",
                              "--deterministic", "true", "--attention", "sdpa", *extra])

    res = warmup(8)
    assert res["executor"] == "FusedLlamaStepper" and res["update_step"] == 8
    assert torch.isfinite(torch.tensor(res["final_eval_loss"]))
    saved = os.path.join(warm, "model_8")
    state = load_state_dict_files(saved)
    module = LlamaForCausalLM(load_config(saved))
    ckpt_lib.load_model_weights(module.to(BF), saved, strict=True)
    assert module.model.layers[0].mlp.down_proj.weight.shape == (256, 341)
    for k, v in module.state_dict().items():
        if not k.endswith("rotary_emb.inv_freq"):
            assert torch.equal(v, state[k].to(v.dtype)), k

    res2 = main(common + ["--use_peft", "--lora_r", "128", "--relora", "4", "--cycle_length", "4",
                               "--restart_warmup_steps", "1", "--scheduler", "cosine_restarts", "--init_lora_a", "kaiming",
                               "--warmed_up_model", saved, "--num_training_steps", "16", "--save_every", "100",
                               "--save_dir", rel])
    assert res2["executor"] == "FusedLlamaStepper" and res2["update_step"] == 16 and res2["n_lora_restarts"] >= 1
    assert torch.isfinite(torch.tensor(res2["final_eval_loss"]))

    res3 = warmup(12, "--autoresume", "true", "--skip_batches", "9")
    assert res3["executor"] == "FusedLlamaStepper" and res3["update_step"] == 12 and "model_12" in os.listdir(warm)
    assert torch.isfinite(torch.tensor(res3["final_eval_loss"]))
