"""`--activation_checkpointing` on the fused executors, on the H100 (-m gpu): for Llama (MHA and GQA) and Pythia (parallel and
sequential residual), bf16 ReLoRA, MXFP8-packed ReLoRA and full-rank training, wgmma and SDPA attention, with and without LoRA
dropout and CUDA graphs, the recompute against save mode on the same weights, ids and dropout seed:

* what each layer's backward reads is byte for byte what save mode kept;
* loss, gradient norm and fp32 gradients of one micro-step, and the parameters after several updates and a merge, differ from save
  mode by no more than save mode differs from itself (split-K, norm and cross-entropy sums use fp32 atomics);
* the peak memory drops by at least 80 % of what the buffer shapes predict."""
import copy
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
DEV = torch.device("cuda", 0)


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, DEV, "nccl")


def _llama(kind, nkv, p, layers, h=256, inter=688, nh=4):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="llama", vocab_size=4096, hidden_size=h, intermediate_size=inter, num_hidden_layers=layers,
                       num_attention_heads=nh, num_key_value_heads=nkv, rms_norm_eps=1e-6, pad_token_id=-1,
                       max_position_embeddings=512)
    torch.manual_seed(0)
    m = LlamaForCausalLM(cfg)
    if kind == "full":
        return m.cuda().to(BF).train()
    w = ReLoRaModel(m, r=128, lora_alpha=32, lora_dropout=p, target_modules=["attn", "mlp"], init_lora_a="kaiming",
                    quantize="mxfp8" if kind == "mx" else None)
    torch.manual_seed(1)
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF).train()


def _pythia(kind, parallel, p, layers, h=256, nh=4):
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=1024, hidden_size=h, num_hidden_layers=layers, num_attention_heads=nh,
                       intermediate_size=4 * h, rotary_pct=0.25, max_position_embeddings=512, layer_norm_eps=1e-5,
                       use_parallel_residual=parallel, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    torch.manual_seed(0)
    m = GPTNeoXForCausalLM(cfg)
    if kind == "full":
        return m.cuda().to(BF).train()
    w = ReLoRaModel(m, r=128, lora_alpha=32, lora_dropout=p, target_modules=["attn", "attention", "mlp"], init_lora_a="kaiming",
                    quantize="mxfp8" if kind == "mx" else None)
    torch.manual_seed(1)
    with torch.no_grad():
        for mod in w.relora_modules():
            torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
            torch.nn.init.normal_(mod.bias, std=0.02)
    return w.cuda().to(BF).train()


def _stepper(arch, model, kind, attention, graphs, ckpt):
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.fused_pythia import FusedPythiaStepper

    cls = FusedLlamaStepper if arch == "llama" else FusedPythiaStepper
    kw = dict(quantize="mxfp8") if kind == "mx" else {}
    return cls(model, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs, attention=attention,
               activation_checkpointing=ckpt, **kw)


def _record_backward_inputs(st):
    """Every slot buffer of layer l as its backward starts (right after the recompute, where there is one)."""
    seen = {}
    recompute = st._recompute

    def hooked(l):
        recompute(l)
        sl = st._slot(l)
        seen[l] = [t[sl].clone() for t in st._slotted]

    st._recompute = hooked
    return seen


def _within(x, ref, ref2, floor, what):
    """|x - ref| within four times save mode's own run-to-run difference |ref2 - ref|, plus ``floor`` for the case where one pair
    of save-mode runs happens to agree bit for bit while the atomics of another run order differently."""
    d, spread = float((x - ref).double().norm()), float((ref2 - ref).double().norm())
    assert d <= 4 * spread + floor, f"{what}: recompute differs by {d:.3e}, save mode from itself by {spread:.3e} (floor {floor:.1e})"


# (arch, kind, shape: nkv for Llama / parallel residual for Pythia, attention, p, graphs, layers)
VARIANTS = [
    ("llama", "bf16", 4, "native", 0.1, False, 4),
    ("llama", "bf16", 4, "native", 0.0, True, 5),
    ("llama", "bf16", 2, "native", 0.1, True, 4),
    ("llama", "bf16", 2, "sdpa", 0.1, False, 4),
    ("llama", "bf16", 4, "sdpa", 0.0, True, 4),
    ("llama", "mx", 4, "native", 0.1, False, 5),
    ("llama", "mx", 2, "sdpa", 0.0, True, 4),
    ("llama", "full", 4, "native", 0.0, False, 4),
    ("llama", "full", 2, "sdpa", 0.0, True, 4),
    ("pythia", "bf16", True, "native", 0.1, False, 4),
    ("pythia", "bf16", False, "native", 0.0, True, 5),
    ("pythia", "bf16", False, "sdpa", 0.1, False, 4),
    ("pythia", "bf16", True, "sdpa", 0.0, True, 4),
    ("pythia", "mx", True, "native", 0.1, True, 4),
    ("pythia", "mx", False, "sdpa", 0.0, False, 4),
    ("pythia", "full", True, "native", 0.0, False, 4),
    ("pythia", "full", False, "sdpa", 0.0, True, 4),
]


@pytest.mark.parametrize("arch,kind,shape,attention,p,graphs,layers", VARIANTS)
def test_recompute_matches_save_mode(arch, kind, shape, attention, p, graphs, layers):
    from relora_b200.ops import fused

    base = _llama(kind, shape, p, layers) if arch == "llama" else _pythia(kind, shape, p, layers)
    models = [copy.deepcopy(base), copy.deepcopy(base), base]
    save, save2, rec = (_stepper(arch, m, kind, attention, graphs, ck) for m, ck in zip(models, (False, False, True)))
    assert rec.recompute and not save.recompute and rec.native_attn == (attention == "native")
    T = 160 if arch == "llama" else 96
    V = base.config.vocab_size if kind == "full" else base.wrapped_model.config.vocab_size
    g = torch.Generator().manual_seed(11)
    ids = [torch.randint(0, V, (2, T), generator=g).to(DEV) for _ in range(4)]
    seen = {} if graphs else {id(st): _record_backward_inputs(st) for st in (save, rec)}
    sts = (save, save2, rec)

    # ---- one micro-step: what each backward reads, then loss and gradients
    losses, grads = [], []
    for st in sts:
        fused.seed_state.set(DEV, 4321)
        losses.append(st.micro_step(ids[0]).double())
        grads.append(st.store.grads.clone())
    assert rec.qkv.shape[0] == 2 and save.qkv.shape[0] == layers
    if seen:
        a, b = seen[id(save)], seen[id(rec)]
        assert sorted(a) == sorted(b) == list(range(layers))
        for l in range(layers):
            for i, (x, y) in enumerate(zip(a[l], b[l])):
                assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"layer {l}, slot buffer {i}: not byte-identical"
    _within(losses[2], losses[0], losses[1], 1e-6 * float(losses[0].abs()), "loss")
    assert float(grads[0].norm()) > 0
    _within(grads[2], grads[0], grads[1], 1e-5 * float(grads[0].norm()), "fp32 gradients")
    norms = [st.update().grad_norm.double() for st in sts]
    _within(norms[2], norms[0], norms[1], 1e-5 * float(norms[0]), "gradient norm")

    # ---- several updates with a merge between them
    p0 = save.store.params.float().clone()
    for step in (1, 2, 3):
        for st in sts:
            fused.seed_state.set(DEV, 100 + step)
            st.micro_step(ids[step])
            st.update()
            if step == 2 and kind != "full":
                st.merge_and_reinit()
    params = [st.store.params.float() for st in sts]
    moved = float((params[0] - p0).norm())
    assert moved > 0
    # AdamW moves an entry whose gradient is near zero by about ±lr, so one sign flip of such a gradient is 2·lr
    _within(params[2], params[0], params[1], 1e-3 * moved, "parameters after 4 updates and a merge")
    evals = [st.eval_loss(ids[0]).double() for st in sts]  # reads the merged frozen weights too
    _within(evals[2], evals[0], evals[1], 1e-4 * float(evals[0].abs()), "evaluation loss after the merge")


@pytest.mark.parametrize("arch", ["llama", "pythia"])
def test_peak_memory_drops_by_the_predicted_amount(arch):
    """Eight layers at 4 x 512 tokens: save mode's peak less the recompute's is at least 80 % of (L - 2) slots of every per-layer
    buffer, the reduction the buffer shapes predict."""
    L = 8
    ids = torch.randint(0, 1024, (4, 512), generator=torch.Generator().manual_seed(0)).to(DEV)
    peaks, predicted = {}, None
    for ck in (False, True):
        model = _llama("bf16", 8, 0.1, L, h=512, inter=1376, nh=8) if arch == "llama" else _pythia("bf16", True, 0.1, L, h=512, nh=8)
        st = _stepper(arch, model, "bf16", "native", False, ck)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        st.micro_step(ids)
        torch.cuda.synchronize()
        peaks[ck] = torch.cuda.max_memory_allocated() - before
        if ck:
            assert st.n_slots == 2
            predicted = (L - 2) * st.saved_bytes_per_layer()
        del st, model
        gc.collect()
        torch.cuda.empty_cache()
    measured = peaks[False] - peaks[True]
    assert measured >= 0.8 * predicted, (measured, predicted, peaks)
