"""`--engine fused --quantize 8bit` on the H100 (-m gpu): the grouped LoRA segment of gemm_mx against the exact reference, the
fused executor on MXFP8-packed stacks against the module path on the same packed bytes and dropout masks, every MXFP8 call of a
micro-step and a merge against the exact contracts, the requantising merge byte for byte, resident memory, and the CLI."""
import copy
import json
import os

import pytest
import torch

from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
LLAMA3 = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 64}


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _tiled(rows, cols, g, tile_rows):
    """bf16 with a power-of-two magnitude of its own per tile_rows x 32 block, so a scale read from the wrong block shows."""
    i = torch.arange(rows, device="cuda").unsqueeze(1) // tile_rows
    j = torch.arange(cols, device="cuda").unsqueeze(0) // 32
    return (torch.randn(rows, cols, generator=g, device="cuda") * torch.exp2(((i + 2 * j) % 5 - 2).float())).to(BF)


# ----------------------------------------------------------------------------------------------- the grouped LoRA segment
@pytest.mark.parametrize("M,G,Ng,K,r,res", [(300, 2, 256, 256, 128, False), (4100, 3, 384, 384, 128, False),
                                             (129, 3, 128, 256, 64, True), (1000, 2, 640, 128, 128, True)])
def test_grouped_lora_segment_matches_the_exact_reference(C, M, G, Ng, K, r, res):
    """out = xq·Wᵀ + u_g·B_gᵀ per group (+ residual), element by element within the fp8 bound; M not a multiple of 128 in the
    ragged cases and more tiles than SMs in the second (the persistent loop)."""
    g = _gen(M + G + Ng)
    N = G * Ng
    xq, sfx = ref.mx_quantize_rows_exact(_tiled(M, K, g, 1))
    wq, sfw, _ = ref.mx_quantize_weight_2d_exact(_tiled(N, K, g, 32))
    u = (torch.randn(M, G * r, generator=g, device="cuda") * 0.5).to(BF)
    B = (torch.randn(N, r, generator=g, device="cuda") * 0.1).to(BF)
    rr = torch.randn(M, N, generator=g, device="cuda").to(BF) if res else None
    out = torch.full((M, N), float("nan"), dtype=BF, device="cuda")
    C.gemm_mx(xq, sfx, wq, sfw, out, M, N, K, False, u, B, rr, Ng, r)
    want, bound = ref.gemm_mx_ref(xq, sfx, wq, sfw, M, N, K, a2=u, b2=B, residual=rr, n_per_group=Ng, a2_group_kofs=r)
    ref.assert_gemm_close(out, want, bound, fp8=True)


def test_gqa_column_windows_match_the_exact_reference(C):
    """The q columns and the k | v columns of a stacked projection under grouped-query attention: two launches into column
    windows of one output, reading windows of the stack's bytes and forward scales."""
    M, h, kv, r = 257, 512, 128, 128
    N = h + 2 * kv
    g = _gen(7)
    xq, sfx = ref.mx_quantize_rows_exact(_tiled(M, h, g, 1))
    wq, sfw, _ = ref.mx_quantize_weight_2d_exact(_tiled(N, h, g, 32))
    u = (torch.randn(M, 3 * r, generator=g, device="cuda") * 0.5).to(BF)
    B = (torch.randn(N, r, generator=g, device="cuda") * 0.1).to(BF)
    out = torch.full((M, N), float("nan"), dtype=BF, device="cuda")
    o = C.mx_sf_bytes(h, h)
    C.gemm_mx(xq, sfx, wq[:h], sfw[:o], out[:, :h], M, h, h, False, u[:, :r], B[:h])
    C.gemm_mx(xq, sfx, wq[h:], sfw[o:], out[:, h:], M, 2 * kv, h, False, u[:, r:], B[h:], None, kv, r)
    base, bound = ref.gemm_mx_ref(xq, sfx, wq, sfw, M, N, h)
    for i, (n0, n1) in enumerate(((0, h), (h, h + kv), (h + kv, N))):
        x, y = u[:, i * r:(i + 1) * r].double(), B[n0:n1].double()
        base[:, n0:n1] += x @ y.t()
        bound[:, n0:n1] += x.abs() @ y.abs().t()
    ref.assert_gemm_close(out, base, bound, fp8=True)


def test_a_group_width_that_is_not_a_multiple_of_128_is_refused(C):
    xq = torch.zeros(128, 128, dtype=torch.uint8, device="cuda")
    sf = torch.zeros(C.mx_sf_bytes(256, 128), dtype=torch.uint8, device="cuda")
    out = torch.empty(128, 192, dtype=BF, device="cuda")
    u, B = torch.zeros(128, 128, dtype=BF, device="cuda"), torch.zeros(192, 64, dtype=BF, device="cuda")
    with pytest.raises(RuntimeError, match="multiple of 128"):
        C.gemm_mx(xq, sf, torch.zeros(256, 128, dtype=torch.uint8, device="cuda"), sf, out, 128, 192, 128, False, u, B, None, 96, 64)


# ----------------------------------------------------------------------------------------------- MX copies of the producers
def _mx_pair(M, K):
    return (torch.full((M, K), 0xA5, dtype=torch.uint8, device="cuda"),
            torch.zeros(ref.mx_sf_bytes(M, K), dtype=torch.uint8, device="cuda"))


def _assert_mx_rows(q, sf, y):
    """q / sf hold the bytes mx_quantize_rows writes for the bf16 y (rows < M; the scales of the padding rows are not written)."""
    M, K = y.shape
    wq, wsf = ref.mx_quantize_rows_exact(y)
    ref.assert_e4m3_bytes_equal("mx q", q, wq)
    ref.assert_bitwise_equal("mx sf", ref.mx_scale_grid(sf, M, K)[:M], ref.mx_scale_grid(wsf, M, K)[:M])


@pytest.mark.parametrize("H", [256, 2048, 4096])  # the warp-per-row kernel, and the block kernel above 2048
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_rmsnorm_emits_the_mx_rows_of_its_output(C, H, p):
    M = 300
    g = _gen(H)
    x = _tiled(M, H, g, 1)
    w = (1 + 0.1 * torch.randn(H, generator=g, device="cuda")).to(BF)
    seed = torch.tensor([12345], dtype=torch.int32, device="cuda")
    G = 2 if p > 0 else 0
    outs = []
    for with_mx in (False, True):
        y, rstd = torch.empty(M, H, dtype=BF, device="cuda"), torch.empty(M, device="cuda")
        xd = torch.empty(M, G * H, dtype=BF, device="cuda") if G else None
        kw = {}
        if with_mx:
            q, sf = _mx_pair(M, H)
            kw = dict(q8=q, q_amax=sf)  # no q_inv_scale: the MX copy
        C.rmsnorm_fwd(x, w, y, rstd, 1e-6, xd, seed if G else None, [3, 4][:G], p, **kw)
        outs.append((y, rstd, xd))
    for a, b in zip(outs[0], outs[1]):  # the outputs the kernel already had are unchanged
        if a is not None:
            assert torch.equal(a, b)
    _assert_mx_rows(q, sf, outs[1][0])


@pytest.mark.parametrize("F", [512, 1408])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_swiglu_emits_the_mx_rows_of_its_output(C, F, p):
    M = 1000
    g = _gen(F)
    gu = (torch.randn(M, 2 * F, generator=g, device="cuda") * 2).to(BF)
    seed = torch.tensor([777], dtype=torch.int32, device="cuda")
    outs = []
    for with_mx in (False, True):
        h = torch.empty(M, F, dtype=BF, device="cuda")
        hd = torch.empty(M, F, dtype=BF, device="cuda") if p > 0 else None
        kw = {}
        if with_mx:
            q, sf = _mx_pair(M, F)
            kw = dict(q8=q, q_amax=sf)  # no q_inv_scale: the MX copy
        C.swiglu_fwd(gu, h, hd, seed if p > 0 else None, 9, p, **kw)
        outs.append((h, hd))
    for a, b in zip(outs[0], outs[1]):
        if a is not None:
            assert torch.equal(a, b)
    _assert_mx_rows(q, sf, outs[1][0])


# ----------------------------------------------------------------------------------------------- the executor
def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _model(p_drop, nkv=4, inter=512, h=256, layers=2, quantize="mxfp8", seed=0):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    kw = dict(rope_theta=500000.0, rope_scaling=dict(LLAMA3)) if nkv != 4 else {}
    cfg = SimpleConfig(model_type="llama", vocab_size=4096, hidden_size=h, intermediate_size=inter, num_hidden_layers=layers,
                       num_attention_heads=4, num_key_value_heads=nkv, rms_norm_eps=1e-6, pad_token_id=-1, max_position_embeddings=256,
                       **kw)
    torch.manual_seed(seed)
    w = ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=p_drop, target_modules=["attn", "mlp"],
                    init_lora_a="kaiming", quantize=quantize)
    torch.manual_seed(seed + 1)
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


def _grads(st):
    return {n: st.store.view_like(st.store.grads, p).float() for n, p in zip(st.trainable_names, st.trainable_params)}


def _ids(B=3, T=128):
    return torch.randint(0, 4096, (B, T), generator=torch.Generator().manual_seed(5)).cuda()


@pytest.mark.parametrize("p_drop,graphs,nkv,inter", [(0.0, False, 4, 512), (0.1, False, 2, 520), (0.0, True, 2, 512),
                                                      (0.1, True, 4, 520)])
def test_fused_mx_matches_the_module_path(p_drop, graphs, nkv, inter):
    """Fused-MX against ModuleStepper on the same packed bytes and dropout masks (MHA and GQA with llama3 RoPE, an intermediate
    size that is not a multiple of 128), then an update, a second step and evaluation."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.engine.stepper import ModuleStepper
    from relora_b200.ops import fused

    wa = _model(p_drop, nkv, inter)
    wb = copy.deepcopy(wa)
    fs = FusedLlamaStepper(wa, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=graphs, quantize="mxfp8")
    ms = ModuleStepper(wb, _info(), lr=1e-3, grad_accumulation=1, native=fused.NativeOptim())
    # the executor's stacks hold the module path's bytes
    for ma, mb in zip(wa.relora_modules(), wb.relora_modules()):
        assert torch.equal(ma.qweight.q, mb.qweight.q) and torch.equal(ma.qweight.sf_fwd, mb.qweight.sf_fwd)
        assert torch.equal(ma.qweight.sf_bwd, mb.qweight.sf_bwd)
    dev = torch.device("cuda", 0)
    ids = _ids()
    fused.seed_state.set(dev, 4321)
    la = fs.micro_step(ids)
    fused.seed_state.set(dev, 4321)
    lb = ms.micro_step(ids)
    assert abs(float(la) - float(lb)) < 4e-2, (float(la), float(lb))
    ga, gb = _grads(fs), _grads(ms)
    for n in ga:
        if gb[n].norm() == 0:
            continue
        e = _relerr(ga[n], gb[n])
        assert e < 0.15, (n, e)
    before = fs.store.params.clone()
    fs.update()
    ms.update()
    assert not torch.equal(before, fs.store.params)
    pa = {n: fs.store.view_like(fs.store.params, p).float() for n, p in zip(fs.trainable_names, fs.trainable_params)}
    pb = {n: ms.store.view_like(ms.store.params, p).float() for n, p in zip(ms.trainable_names, ms.trainable_params)}
    pa0 = {n: fs.store.view_like(before, p).float() for n, p in zip(fs.trainable_names, fs.trainable_params)}
    for n in pa:  # AdamW's first step moves each entry by about lr·sign(g): entries with gradients near zero may flip, so the
        da, db = (pa[n] - pa0[n]).flatten(), (pb[n] - pa0[n]).flatten()  # steps are compared by direction
        if db.norm() > 0:
            cos = float(torch.dot(da, db) / (da.norm() * db.norm()))
            assert cos > 0.9, (n, cos)
    l2 = fs.micro_step(ids)
    assert torch.isfinite(l2)
    ev, evm = fs.eval_loss(ids), ms.eval_loss(ids)
    assert torch.isfinite(ev) and abs(float(ev) - float(evm)) < 4e-2, (float(ev), float(evm))


class _Audit:
    """Checks every MXFP8 call against the exact contract of ops/reference.py and records each merge's delta."""

    def __init__(self, C, monkeypatch):
        self.C, self.modes, self.deltas = C, {}, []
        self.orig = {n: getattr(C, n) for n in ("mx_quantize_rows", "gemm_mx", "mx_quantize_weight_2d")}
        for n in self.orig:
            monkeypatch.setattr(C, n, (lambda name: lambda *a: self.call(name, *a))(n))

    def call(self, name, *a):
        torch.cuda.synchronize()
        b = [x.clone() if torch.is_tensor(x) else x for x in a]
        self.orig[name](*a)
        torch.cuda.synchronize()
        mode = getattr(self, "_" + name)(b, a)
        self.modes[mode] = self.modes.get(mode, 0) + 1

    def _mx_quantize_rows(self, b, a):
        x, q, sf = b[0], a[1], a[2]
        wq, wsf = ref.mx_quantize_rows_exact(x)
        ref.assert_e4m3_bytes_equal("mx_quantize_rows q", q[:, :wq.shape[1]], wq)
        ref.assert_bitwise_equal("mx_quantize_rows sf", sf[:wsf.numel()], wsf)
        return "quantize_rows"

    def _gemm_mx(self, b, a):
        xa, sfa, wb, sfb, _, M, N, K, mn = b[:9]
        a2, b2, res = (list(b[9:12]) + [None] * 3)[:3]
        npg, kofs = (list(b[12:14]) + [0, 0])[:2]
        want, bound = ref.gemm_mx_ref(xa, sfa, wb, sfb, M, N, K, mn, a2, b2, res, n_per_group=npg, a2_group_kofs=kofs)
        ref.assert_gemm_close(a[4][:M, :N], want, bound, fp8=True)
        return f"gemm_mx {'MN' if mn else 'K'}-major{' LoRA' if a2 is not None else ''}{' grouped' if npg else ''}" \
               f"{' residual' if res is not None else ''}"

    def _mx_quantize_weight_2d(self, b, a):
        w, delta, q_old, f_old, _, N, K = b
        assert w is None, "the executor only requantises"
        self.deltas.append(delta)
        q, f, bw = ref.mx_quantize_weight_2d_exact(q_old=q_old, sf_old=f_old, delta=delta, N=N, K=K)
        ref.assert_e4m3_bytes_equal("merge q", a[2][:q.shape[0], :q.shape[1]], q)
        ref.assert_bitwise_equal("merge sf_fwd", a[3][:f.numel()], f)
        ref.assert_bitwise_equal("merge sf_bwd", a[4][:bw.numel()], bw)
        return "merge"


def test_every_mx_call_of_a_micro_step_and_a_merge_matches_the_contract(C, monkeypatch):
    """One fused micro-step (dropout, grouped-query attention, padded intermediate size) and one merge: every MXFP8 call
    checked; the merge's requantised bytes, which each module's packed weight aliases, are the exact requantisation of the old
    bytes plus the executor's delta, and that delta is s·B·A."""
    from relora_b200.engine.fused_llama import FusedLlamaStepper
    from relora_b200.ops import fused, mx

    w = _model(0.1, nkv=2, inter=520)
    fs = FusedLlamaStepper(w, _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False, quantize="mxfp8")
    mods = list(w.relora_modules())
    old = [(m.qweight.q.clone(), m.qweight.sf_fwd.clone()) for m in mods]
    AB = [(m.lora_A.weight.detach().float().clone(), m.lora_B.weight.detach().float().clone()) for m in mods]
    audit = _Audit(C, monkeypatch)
    fused.seed_state.set(torch.device("cuda", 0), 77)
    fs.micro_step(_ids())
    fs.merge_and_reinit()
    torch.cuda.synchronize()
    print(f"[fused mx audit] {dict(sorted(audit.modes.items()))}")
    L = len(fs.layers)
    assert audit.modes["merge"] == 4 * L
    assert {"quantize_rows", "gemm_mx K-major LoRA", "gemm_mx K-major LoRA grouped", "gemm_mx K-major LoRA residual",
            "gemm_mx MN-major"} <= set(audit.modes)
    # the norms and SwiGLU emit the MX rows of qkv, gate|up and down: only the attention output (o) and the 4 backward dy are
    # quantised by mx_quantize_rows
    assert audit.modes["quantize_rows"] == 5 * L
    # each module's rows of its stack's delta, and its bytes after the merge
    s = fs.scale
    for l in range(L):
        rows = fs._stack_rows(w.wrapped_model.model.layers[l])
        for gi, group in enumerate(rows):
            d = audit.deltas[4 * l + gi]
            for m, r0 in group:
                i = mods.index(m)
                A, B = AB[i]
                dm = d[r0:r0 + m.out_features, :m.in_features]
                assert _relerr(dm, s * (B @ A)) < 1e-5
                q, f, bw = ref.mx_quantize_weight_2d_exact(q_old=old[i][0], sf_old=old[i][1], delta=dm, N=m.out_features,
                                                           K=m.in_features)
                ref.assert_e4m3_bytes_equal("module q", m.qweight.q[:q.shape[0], :q.shape[1]], q)
                ref.assert_bitwise_equal("module sf_fwd", m.qweight.sf_fwd, f)
                ref.assert_bitwise_equal("module sf_bwd", m.qweight.sf_bwd, bw)
                assert m.qweight.q.data_ptr() == fs.Wmx[l][gi].q[r0].data_ptr()
    assert isinstance(mods[0].qweight, mx.MxWeight)


def test_packed_stacks_are_the_only_resident_frozen_weights():
    """No bf16 frozen stack exists, and the device memory after construction is below the bf16 executor's on the same model by
    at least 90 % of the bytes packing saves."""
    import gc

    from relora_b200.engine.fused_llama import FusedLlamaStepper

    def build(quantize):
        gc.collect()
        torch.cuda.empty_cache()
        m = _model(0.0, h=512, inter=1376, layers=4, quantize=quantize)
        fs = FusedLlamaStepper(m, _info(), lr=1e-3, cuda_graphs=False, quantize=quantize)
        torch.cuda.synchronize()
        return m, fs, torch.cuda.memory_allocated()

    m, fs, bf16_bytes_alloc = build(None)
    frozen_bf16 = sum(t.numel() * 2 for t in (fs.Wqkv, fs.Wo, fs.Wgu, fs.Wd))
    del m, fs
    m, fs, mx_alloc = build("mxfp8")
    assert fs.Wqkv is None and fs.Wo is None and fs.Wgu is None and fs.Wd is None
    packed = sum(st.nbytes for stacks in fs.Wmx for st in stacks)
    for mod in m.relora_modules():
        assert "weight" not in mod._parameters and mod.qweight.q.dtype == torch.uint8
    saved = bf16_bytes_alloc - mx_alloc
    print(f"[fused mx memory] bf16 executor {bf16_bytes_alloc / 2**20:.1f} MiB, mx {mx_alloc / 2**20:.1f} MiB, "
          f"frozen bf16 {frozen_bf16 / 2**20:.1f} MiB, packed {packed / 2**20:.1f} MiB")
    assert saved >= 0.9 * (frozen_bf16 - packed), (saved, frozen_bf16, packed)


# ----------------------------------------------------------------------------------------------- command line
def _cli_args(tmp_path, quant, steps=8):
    cfg = {"architectures": ["LlamaForCausalLM"], "model_type": "llama", "vocab_size": 4096, "hidden_size": 256, "intermediate_size": 512,
           "num_hidden_layers": 2, "num_attention_heads": 4, "num_key_value_heads": 2, "rms_norm_eps": 1e-6, "max_sequence_length": 256,
           "hidden_act": "silu", "bos_token_id": 0, "eos_token_id": 1, "pad_token_id": -1, "initializer_range": 0.02, "use_cache": True}
    cfg_path = str(tmp_path / "llama_tiny.json")
    json.dump(cfg, open(cfg_path, "w"))
    return ["--model_config", cfg_path, "--synthetic_data", "4096", "--batch_size", "4", "--total_batch_size", "8", "--max_length", "128",
            "--lr", "1e-3", "--use_peft", "--lora_r", "128", "--relora", "4", "--cycle_length", "4", "--restart_warmup_steps", "1",
            "--scheduler", "cosine_restarts", "--warmup_steps", "2", "--num_training_steps", str(steps), "--save_every", "4",
            "--eval_every", "100", "--save_dir", str(tmp_path / "run"), "--dtype", "bfloat16", "--workers", "0", "--init_lora_a",
            "kaiming", "--quantize", quant, "--engine", "fused"]


def test_cli_fused_8bit_restarts_checkpoints_and_resumes(tmp_path):
    from torchrun_main import main

    args = _cli_args(tmp_path, "8bit")
    res = main(args)
    assert res["executor"] == "FusedLlamaStepper" and res["update_step"] == 8 and res["n_lora_restarts"] == 1
    assert torch.isfinite(torch.tensor(res["final_eval_loss"])) and res["final_eval_loss"] < 9.0
    sd = torch.load(os.path.join(str(tmp_path / "run"), "model_8", "pytorch_model.bin"), weights_only=True)
    for k in ("model.layers.0.self_attn.q_proj.weight", "model.layers.0.self_attn.k_proj.weight", "model.layers.1.mlp.down_proj.weight"):
        w = sd[k]
        assert w.dim() == 2 and w.dtype == BF and bool(torch.isfinite(w.float()).all()), k
    assert sd["model.layers.0.self_attn.k_proj.weight"].shape == (128, 256)
    res2 = main(args[:args.index("--num_training_steps")] + ["--num_training_steps", "12"] +
                args[args.index("--num_training_steps") + 2:] + ["--autoresume", "true"])
    assert res2["executor"] == "FusedLlamaStepper" and res2["update_step"] == 12
    assert "model_12" in os.listdir(str(tmp_path / "run"))


def test_cli_fused_4bit_is_refused_with_its_reason(tmp_path):
    from torchrun_main import main

    with pytest.raises(RuntimeError, match="only 8bit \\(mxfp8\\) frozen weights run on the fused executor"):
        main(_cli_args(tmp_path, "4bit"))
