"""Every addressing and epilogue mode of the wgmma GEMM (csrc/gemm_wgmma.cu) and the fused LoRA input-gradient kernel, element
by element against the fp64 reference of their contract (ops/reference.py: gemm_ref, lora_dx_ref, assert_gemm_close), and an
audit of every such call the fused executors issue (H100: -m gpu).

Operands sit inside larger NaN-filled buffers (row pitch above the width, extra rows above and below): a kernel that reads past
the extents it was given picks up a NaN.  Outputs sit inside buffers whose guard region holds a sentinel that must survive bit
for bit, and their interior starts as NaN unless the call accumulates, so an element that is never written fails too."""
import math

import pytest
import torch

from gemm_forms import FORMS, lora_group_call, lora_group_shapes
from guarded_buffers import Guarded
from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF, F32 = torch.bfloat16, torch.float32
M_TOK, K_H, R = 291, 256, 128
SENTINEL = 1234.0
WORST = {}  # worst error/tolerance ratio per case family (printed at the end of the module with -s)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for fam, (w, case) in sorted(WORST.items()):
        print(f"[gemm modes] {fam}: worst ratio {w:.3g} ({case})")


def _note(family, worst, case):
    if worst > WORST.get(family, (-1.0, ""))[0]:
        WORST[family] = (worst, case)


@pytest.fixture(scope="module")
def F():
    from relora_b200.ops import fused

    fused._C()
    return fused


def _Buf(src, fill, interior=None):
    # pitch a multiple of 16 elements: every row start stays 16-byte aligned for the one-byte fp8 operands too
    return Guarded(src, fill, interior, pitch_multiple=16)


def _operand(t):
    return _Buf(t, 0x7F if t.dtype == torch.uint8 else float("nan")).view  # 0x7F: NaN in E4M3 and E5M2


def _output(t, accumulate):
    return _Buf(t, SENTINEL, interior=None if accumulate else torch.full_like(t, float("nan")))


def _rand(*shape, scale=1.0, dtype=BF, seed=None):
    if seed is not None:
        torch.manual_seed(seed)
    return (torch.randn(*shape, device="cuda") * scale).to(dtype)


def _check(F, family, case, a1, b1, out_t, **kw):
    """gemm on guarded copies of the operands / output, guards checked, result against gemm_ref."""
    acc = bool(kw.get("accumulate", False))
    ops = {k: (_operand(v) if torch.is_tensor(v) and k != "alpha_dev" else v) for k, v in kw.items()}
    o = _output(out_t, acc)
    prev = o.view.clone()
    A1, B1 = _operand(a1), _operand(b1)
    F.gemm(A1, B1, o.view, **ops)
    torch.cuda.synchronize()
    assert o.guards_intact(), f"{case}: the output guard region was written"
    want, bound = ref.gemm_ref(A1, B1, prev, **ops)
    w = ref.assert_gemm_close(o.view, want, bound, fp8=bool(kw.get("fp8", 0)))
    _note(family, w, case)
    if o.view.dtype == F32:  # no output rounding to speak of: the accumulation error itself, per unit of the bound
        _note(family + " fp32 |err|/bound", float(((o.view.double() - want).abs() / bound.clamp(min=1e-300)).max()), case)
    return o.view


# ----------------------------------------------------------------------------------------------- plain, both majors
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M", [1, 129])
@pytest.mark.parametrize("N", [129, 1001])
@pytest.mark.parametrize("K", [8, 72])
def test_plain(F, M, N, K, a_mn, b_mn):
    a, b = _rand(M, K, seed=M + N + K), _rand(N, K, scale=0.05)
    _check(F, "bf16 plain", f"M={M} N={N} K={K} mn={a_mn},{b_mn}", a.t().contiguous() if a_mn else a,
           b.t().contiguous() if b_mn else b, torch.empty(M, N, dtype=BF, device="cuda"), M=M, N=N, K1=K, a1_mn=a_mn, b1_mn=b_mn)


# ----------------------------------------------------------------------------------------------- bias epilogue
@pytest.mark.parametrize("block_n", [128, 256, 0])
@pytest.mark.parametrize("variant", ["alone", "alpha", "residual", "grouped", "ragged_group"])
def test_bias(F, variant, block_n):
    M, K = M_TOK, K_H
    G, Ng = {"grouped": (3, 256), "ragged_group": (2, 320)}.get(variant, (1, 768))
    N = G * Ng
    torch.manual_seed(7)
    x, W, bias = _rand(M, K), _rand(N, K, scale=0.05), _rand(N, scale=0.1)
    kw = dict(M=M, N=N, K1=K, bias=bias, block_n=block_n)
    if variant == "alpha":
        kw["alpha"] = 0.37
    if variant in ("residual", "ragged_group"):
        kw["residual"] = _rand(M, N)
    if G > 1:
        kw.update(a2=_rand(M, G * R), b2=_rand(N, R, scale=0.05), K2=R, n_per_group=Ng, a2_group_kofs=R)
    _check(F, "bf16 bias", f"{variant} block_n={block_n}", x, W, torch.empty(M, N, dtype=BF, device="cuda"), **kw)


@pytest.mark.parametrize("extra", ["bias", "residual"])
def test_bias_and_residual_need_a_bf16_output(F, extra):
    """Both are fused into the bf16 epilogue only; an fp32 output would silently drop them, so the call is refused."""
    a, b = _rand(256, 128), _rand(256, 128)
    t = _rand(256) if extra == "bias" else _rand(256, 256)
    with pytest.raises(RuntimeError, match="bf16 output"):
        F.gemm(a, b, torch.zeros(256, 256, dtype=F32, device="cuda"), **{extra: t})


# ----------------------------------------------------------------------------------------------- LoRA group forms
def _group_case(F, form, G, Ng, drop, *, K=K_H, M=M_TOK, split_k=0, family="bf16 lora forms", seed=0):
    dims = dict(G=G, K=K, Ng=Ng, r=R)
    torch.manual_seed(seed)
    T = {}
    for name, (shape, dt) in lora_group_shapes(M=M, drop=drop, **dims).items():
        scale = 0.05 if name in ("A", "W", "B") else (0.1 if name == "bias" else 1.0)
        T[name] = _rand(*shape, scale=scale, dtype=dt)
    a1, b1, out, kw = lora_group_call(form, T, M=M, s=0.25, drop=drop, split_k=split_k, **dims)
    _check(F, family, f"{form} G={G} Ng={Ng} K={K} M={M} drop={drop} split_k={split_k}", a1, b1, out, **kw)


@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("G,Ng", [(1, 256), (2, 384), (3, 256)])
@pytest.mark.parametrize("form", FORMS)
def test_lora_group_forms(F, form, G, Ng, drop):
    """u, y (bias + residual), du, parts, dA (B1 MN offset 0 or K per m-group) and dB as the executors issue them."""
    _group_case(F, form, G, Ng, drop, seed=G)


@pytest.mark.parametrize("split_k", [1, 0, 7])
@pytest.mark.parametrize("form", ["dA", "dB"])
def test_weight_gradients_split_k(F, form, split_k):
    """fp32 weight gradients accumulated onto a non-zero gradient, with and without split-K, grouped (G = 3)."""
    _group_case(F, form, 3, 256, True, split_k=split_k, family="bf16 split-k", seed=11)


@pytest.mark.parametrize("form,G,K,Ng", [("dA", 3, 2048, 2048), ("dB", 2, 2048, 5504)])
def test_weight_gradients_more_work_than_sms(F, form, G, K, Ng):
    """llama_1b-sized weight gradients over 4098 tokens at split_k = 7: tiles × splits well above the SM count."""
    _group_case(F, form, G, Ng, True, K=K, M=4098, split_k=7, family="bf16 split-k", seed=12)


def test_fused_lora_forward_at_llama_1b_gate_up(F):
    """y = [xn | u]·[W | B]ᵀ with two ragged 5504-wide groups (llama_1b gate / up) over 4098 tokens."""
    _group_case(F, "y", 2, 5504, True, K=2048, M=4098, family="bf16 lora forms", seed=13)


# ----------------------------------------------------------------------------------------------- output dtypes, alpha_dev
@pytest.mark.parametrize("mode", ["f32_overwrite", "bf16_accumulate", "alpha_dev_bf16"])
def test_epilogue_modes(F, mode):
    M, N, K = M_TOK, 384, 320
    torch.manual_seed(21)
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    if mode == "f32_overwrite":
        _check(F, "bf16 epilogue", mode, a, b, torch.empty(M, N, dtype=F32, device="cuda"), M=M, N=N, K1=K, alpha=0.5)
    elif mode == "bf16_accumulate":
        _check(F, "bf16 epilogue", mode, a, b, _rand(M, N), M=M, N=N, K1=K, alpha=2.0, accumulate=True)
    else:
        dev = torch.tensor([0.3], dtype=F32, device="cuda")
        _check(F, "bf16 epilogue", mode, a, b, torch.empty(M, N, dtype=BF, device="cuda"), M=M, N=N, K1=K, alpha=1.5,
               alpha_dev=dev, a2=_rand(M, R), b2=_rand(N, R, scale=0.05), K2=R)


# ----------------------------------------------------------------------------------------------- fp8
def _quant(x, dtype):
    s = float(x.float().abs().max()) / torch.finfo(dtype).max
    return (x.float() / s).to(dtype).view(torch.uint8), s


@pytest.mark.parametrize("K", [256, 320])
def test_fp8_e4m3_with_bf16_lora_residual_alpha_dev(F, K):
    """fp8=1: E4M3 x·Wᵀ sharing the accumulator with the bf16 LoRA segment (pre-divided by the product scale), residual."""
    M, N = M_TOK, 768
    torch.manual_seed(K)
    (x8, sx), (w8, sw) = _quant(_rand(M, K), torch.float8_e4m3fn), _quant(_rand(N, K, scale=0.05), torch.float8_e4m3fn)
    alpha = torch.tensor([sx * sw], dtype=F32, device="cuda")
    u = (_rand(M, R).float() / (sx * sw)).to(BF)
    B = _rand(N, R, scale=0.05)
    _check(F, "fp8", f"fp8=1 K={K}", x8, w8, torch.empty(M, N, dtype=BF, device="cuda"), M=M, N=N, K1=K, a2=u,
           b2=B, K2=R, residual=_rand(M, N), fp8=1, alpha_dev=alpha)
    _check(F, "fp8", f"fp8=1 K={K} fp32 out", x8, w8, torch.empty(M, N, dtype=F32, device="cuda"), M=M, N=N, K1=K, a2=u,
           b2=B, K2=R, fp8=1, alpha_dev=alpha)


@pytest.mark.parametrize("Kb", [768, 704])
def test_fp8_e5m2_gradient_times_e4m3_weight(F, Kb):
    """fp8=2 (the fp8_full input gradient): E5M2 dy [M, Kb] × E4M3 Wᵀ [N, Kb]."""
    M, N = M_TOK, K_H
    torch.manual_seed(Kb)
    (d8, sd), (w8, sw) = _quant(_rand(M, Kb), torch.float8_e5m2), _quant(_rand(N, Kb, scale=0.05), torch.float8_e4m3fn)
    for odt in (BF, F32):
        _check(F, "fp8", f"fp8=2 Kb={Kb} {odt}", d8, w8, torch.empty(M, N, dtype=odt, device="cuda"), M=M, N=N, K1=Kb, fp8=2,
               alpha_dev=torch.tensor([sd * sw], dtype=F32, device="cuda"))


# ----------------------------------------------------------------------------------------------- lora_dx
@pytest.mark.parametrize("with_base", [False, True])
@pytest.mark.parametrize("G,Ng,N,M", [(1, 2048, 5504, M_TOK), (2, 5504, 2048, M_TOK), (3, 256, 256, 129), (3, 2048, 2048, 4098)])
def test_lora_dx(F, G, Ng, N, M, with_base):
    C, p, keys = F._C(), 0.1, [11, 22, 33][:G]
    torch.manual_seed(G * 31 + N)
    dy, W, du, A = _operand(_rand(M, G * Ng)), _operand(_rand(G * Ng, N, scale=0.05)), _operand(_rand(M, G * R)), _operand(_rand(G * R, N, scale=0.05))
    base = _operand(_rand(M, N)) if with_base else None
    seed = torch.tensor([1234567], dtype=torch.int32, device="cuda")
    o = _output(torch.empty(M, N, dtype=BF, device="cuda"), False)
    if with_base:
        C.lora_dx(None, None, du, A, o.view, seed, keys, p, base)
    else:
        C.lora_dx(dy, W, du, A, o.view, seed, keys, p)
    torch.cuda.synchronize()
    assert o.guards_intact()
    want, bound = ref.lora_dx_ref(None if with_base else dy, None if with_base else W, du, A, seed, keys, p, base=base)
    _note("lora_dx", ref.assert_gemm_close(o.view, want, bound), f"G={G} Ng={Ng} N={N} M={M} base={with_base}")


# ----------------------------------------------------------------------------------------------- windowed K overhang
def test_windowed_k_not_a_multiple_of_the_k_block(F):
    """du form with G = 2 and Ng = 96: both operands take a per-group K window 96 wide, so group 0's second 64-wide k-block
    runs 32 columns into group 1's window.  The call must either compute the right result or be refused."""
    G, Ng, M = 2, 96, M_TOK
    torch.manual_seed(31)
    dy, B = _rand(M, G * Ng), _rand(G * Ng, R, scale=0.05)
    kw = dict(M=M, N=G * R, K1=Ng, b1_mn=True, n_per_group=R, a1_group_kofs=Ng, b1_group_kofs=Ng, b1_local_n=True, alpha=0.25)
    out = torch.empty(M, G * R, dtype=BF, device="cuda")
    try:
        F.gemm(dy, B, out, **kw)
    except RuntimeError as e:
        assert "multiple of the k-block" in str(e)
        return
    torch.cuda.synchronize()
    want, bound = ref.gemm_ref(dy, B, out, **kw)
    err = float((out.double() - want).abs().max())
    print(f"[gemm modes] windowed-K overhang: max |out - ref| {err:.4g}, max |ref| {float(want.abs().max()):.4g}")
    ref.assert_gemm_close(out, want, bound)


def test_windowed_k_on_one_side_only_is_exact(F):
    """A K window 96 wide on one operand only: u form (A1 windowed, B1 not) and the LoRA segment of y (A2 windowed, B2
    never is).  The overhang meets the other operand's zero fill, so both products are right and neither call is refused."""
    G, K, M = 2, 96, M_TOK
    torch.manual_seed(32)
    _check(F, "bf16 lora forms", "u G=2 K=96", _rand(M, G * K), _rand(G * R, K, scale=0.05), torch.empty(M, G * R, dtype=BF, device="cuda"),
           M=M, N=G * R, K1=K, n_per_group=R, a1_group_kofs=K, alpha=0.25)
    Ng = 256
    _check(F, "bf16 lora forms", "y G=2 K2=96", _rand(M, K_H), _rand(G * Ng, K_H, scale=0.05), torch.empty(M, G * Ng, dtype=BF, device="cuda"),
           M=M, N=G * Ng, K1=K_H, a2=_rand(M, G * K), b2=_rand(G * Ng, K, scale=0.05), K2=K, n_per_group=Ng, a2_group_kofs=K)


# ----------------------------------------------------------------------------------------------- executor audit
class _Audit:
    """Wraps ``fused.gemm`` and the extension's ``lora_dx``: every call is checked against the reference on clones of its
    inputs (taken after a device synchronise: the weight gradients run on a side stream), and its modes are collected."""

    def __init__(self, fused, C):
        self.gemm0, self.dx0 = fused.gemm, C.lora_dx
        self.modes, self.calls, self.worst = set(), 0, 0.0

    def gemm(self, a1, b1, out=None, **kw):
        torch.cuda.synchronize()
        cl = lambda v: v.clone() if torch.is_tensor(v) else v  # noqa: E731
        a1c, b1c, kwc, prev = cl(a1), cl(b1), {k: cl(v) for k, v in kw.items()}, cl(out)
        res = self.gemm0(a1, b1, out, **kw)
        torch.cuda.synchronize()
        want, bound = ref.gemm_ref(a1c, b1c, prev, **kwc)
        self.worst = max(self.worst, ref.assert_gemm_close(res, want, bound, fp8=bool(kw.get("fp8", 0))))
        self.calls += 1
        M = kw.get("M") or (a1.shape[1] if kw.get("a1_mn") else a1.shape[0])
        N = kw.get("N") or (b1.shape[1] if kw.get("b1_mn") else b1.shape[0])
        for k in ("bias", "residual", "alpha_dev"):
            if kw.get(k) is not None:
                self.modes.add(k)
        if math.ceil(N / (kw.get("n_per_group") or N)) > 1:
            self.modes.update(k for k in ("a1_group_kofs", "a2_group_kofs", "b1_group_kofs", "b1_local_n") if kw.get(k))
        if kw.get("m_per_group") and math.ceil(M / kw["m_per_group"]) > 1:
            self.modes.add("m_per_group")
            if kw.get("b1_mn_ofs_per_mgroup"):
                self.modes.add("b1_mn_ofs_per_mgroup")
        if kw.get("split_k", 1) != 1:
            self.modes.add("split_k")
        if kw.get("fp8"):
            self.modes.add(f"fp8={int(kw['fp8'])}")
        return res

    def lora_dx(self, dy, w, du, a, out, seed, keys, p, base=None):
        torch.cuda.synchronize()
        cl = lambda v: v.clone() if torch.is_tensor(v) else v  # noqa: E731
        args = [cl(v) for v in (dy, w, du, a, seed)] + [list(keys), float(p), cl(base)]
        self.dx0(dy, w, du, a, out, seed, keys, p, base)
        torch.cuda.synchronize()
        dyc, wc, duc, ac, sc, ks, pp, bc = args
        want, bound = ref.lora_dx_ref(dyc, wc, duc, ac, sc, ks, pp, base=bc)
        self.worst = max(self.worst, ref.assert_gemm_close(out, want, bound))
        self.calls += 1
        self.modes.add("lora_dx" if base is None else "lora_dx_base")

    def install(self, monkeypatch, fused, C):
        monkeypatch.setattr(fused, "gemm", self.gemm)
        monkeypatch.setattr(C, "lora_dx", self.lora_dx)


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _llama(p_drop, inter):
    from relora_b200.models import LlamaForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="llama", vocab_size=4096, hidden_size=256, intermediate_size=inter, num_hidden_layers=2,
                       num_attention_heads=4, rms_norm_eps=1e-6, pad_token_id=-1, max_position_embeddings=256)
    torch.manual_seed(0)
    w = ReLoRaModel(LlamaForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=p_drop, target_modules=["attn", "mlp"], init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


def _pythia(parallel):
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=1024, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                       intermediate_size=1024, rotary_pct=0.25, max_position_embeddings=64, layer_norm_eps=1e-5,
                       use_parallel_residual=parallel, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    torch.manual_seed(0)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming")
    with torch.no_grad():
        for mod in w.relora_modules():
            torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
            torch.nn.init.normal_(mod.bias, std=0.02)
    return w.cuda().to(BF).train()


_GROUPED = {"residual", "a1_group_kofs", "a2_group_kofs", "b1_group_kofs", "b1_local_n", "m_per_group", "b1_mn_ofs_per_mgroup", "split_k"}
_AUDIT = {
    "llama": _GROUPED | {"lora_dx"},
    "llama_parts": _GROUPED,
    "llama_dx_base": _GROUPED | {"lora_dx_base"},
    "llama_fp8_full": _GROUPED | {"lora_dx_base", "fp8=1", "fp8=2", "alpha_dev"},
    "pythia_parallel": {"bias", "residual", "split_k", "lora_dx"},
    "pythia_sequential": {"bias", "residual", "split_k", "lora_dx"},
}


@pytest.mark.parametrize("config", list(_AUDIT))
def test_executor_gemms_match_the_reference(config, monkeypatch):
    """One training micro-step and one evaluation of each executor configuration, every GEMM and lora_dx call audited
    (CUDA graphs off, 3 x 97 tokens).  The set of modes seen must be the expected one: a path that starts using another
    mode shows up here."""
    from relora_b200.ops import fused

    C = fused._C()
    if config == "llama_parts":
        monkeypatch.setenv("RELORA_B200_FUSED_DX", "0")  # parts GEMM + dropout_combine
    if config in ("llama_dx_base", "llama_fp8_full"):
        monkeypatch.setenv("RELORA_B200_DX_SPLIT_K", "256")  # the two-kernel input gradient (lora_dx with Kb == 0) everywhere
    if config.startswith("pythia"):
        from relora_b200.engine.fused_pythia import FusedPythiaStepper

        st = FusedPythiaStepper(_pythia(config == "pythia_parallel"), _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False)
    else:
        from relora_b200.engine.fused_llama import FusedLlamaStepper

        fp8 = config == "llama_fp8_full"
        st = FusedLlamaStepper(_llama(0.1, 341), _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False, fp8=fp8,
                               fp8_backward=fp8)
    dev = torch.device("cuda", 0)
    ids = torch.randint(0, 1024, (3, 97), device=dev)
    fused.seed_state.set(dev, 4321)
    if config == "llama_fp8_full":
        st.micro_step(ids)  # calibrates the activation scales; the first backward runs in bf16 and records the gradient scales
    audit = _Audit(fused, C)
    audit.install(monkeypatch, fused, C)
    loss = st.micro_step(ids)
    ev = st.eval_loss(ids)
    assert torch.isfinite(loss) and torch.isfinite(ev)
    print(f"[gemm modes] audit {config}: {audit.calls} calls, worst ratio {audit.worst:.3g}, modes {sorted(audit.modes)}")
    _note("audit fp8" if config == "llama_fp8_full" else "audit", audit.worst, config)
    assert audit.modes == _AUDIT[config]
