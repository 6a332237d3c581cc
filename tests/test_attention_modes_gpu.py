"""The wgmma attention kernels (csrc/attention.cu) element by element against the fp64 reference of their contract
(ops/reference.py: attention_ref, assert_attention_close) over every step-count branch and output split, sequence tails that run
into the next batch, grouped-query and interleaved layouts and the score regimes where online softmax goes wrong; and an audit of
every attention call the fused executors and the module path issue (H100: -m gpu).

qkv and dout sit inside larger NaN-filled buffers (row pitch a multiple of 8 elements above the width, a 16-column offset,
NaN rows above and below): a TMA map whose extents are wrong reads a NaN.  out, lse, delta and dqkv sit inside buffers whose
guard region holds a sentinel that must survive bit for bit, and their interior starts as NaN, so an element that is never
written fails too."""
import math

import pytest
import torch

from guarded_buffers import Guarded
from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF, F32 = torch.bfloat16, torch.float32
SENTINEL = 1234.0
WORST = {}  # worst error/tolerance ratio per case family and tensor (printed at the end of the module with -s)
CALIB = {}  # lse error per unit of each tolerance term, for setting ATTN_C_L / ATTN_C_S


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for fam, (w, case) in sorted(WORST.items()):
        print(f"[attention modes] {fam}: worst ratio {w:.3g} ({case})")
    for what, (w, case) in sorted(CALIB.items()):
        print(f"[attention modes] calibration {what}: {w:.3g} ({case})")


def _note(table, family, worst, case):
    if worst > table.get(family, (-1.0, ""))[0]:
        table[family] = (worst, case)


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


def _operand(t):
    return Guarded(t, float("nan"), pitch_multiple=8).view


def _output(t):
    return Guarded(t, SENTINEL, interior=torch.full_like(t, float("nan")), pitch_multiple=8)


REGIMES = ("random", "uniform", "peaked", "rising", "sink", "large", "do_eq_o")


def _qkv(B, T, nh, hd, nkv, interleaved, regime, scale, seed, batch_scale):
    """fp32 packed qkv [B*T, W] of one score regime (rounded to bf16 by the caller)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * T, (nh + 2 * nkv) * hd, generator=g, device="cuda")
    q, k, v = ref.attention_unpack(x, B, T, nh, hd, nkv=nkv, interleaved=interleaved)  # views into x
    if batch_scale:  # every batch at its own scale, so a row that leaks into the next batch is far off
        v.mul_(1.0 + 3.0 * torch.arange(B, device="cuda").view(B, 1, 1, 1))
    if regime == "uniform":  # q = 0: P = 1/(i+1) exactly, O the running mean of v, lse = log2(i+1)
        q.zero_()
    elif regime == "peaked":  # score std ~10 nats
        q.mul_(10.0 ** 0.5 / (scale * hd ** 0.5) ** 0.5)
        k.mul_(10.0 ** 0.5 / (scale * hd ** 0.5) ** 0.5)
    elif regime == "rising":  # each 64-key block raises every row's maximum by 8 nats: corr fires each block, old sums underflow
        q.mul_(0.3)
        k.mul_(0.3)
        q[..., 0] = 1.0
        k[..., 0] = torch.arange(T, device="cuda", dtype=F32) * (8.0 / (64 * scale))
    elif regime == "sink":  # key 0 of each sequence takes ~30 nats over the rest
        q[..., 0] = 1.0
        k[:, :, 0, 0] = 30.0 / scale
    elif regime == "large":  # |s| into the hundreds
        q.mul_(10.0 / (scale * hd ** 0.5) ** 0.5)
        k.mul_(10.0 / (scale * hd ** 0.5) ** 0.5)
    return x.to(BF)


def _case(C, family, B, T, nh, hd, nkv=-1, interleaved=False, scale=None, regime="random", seed=0, batch_scale=False, ws=None):
    """Forward and backward on guarded buffers, guards checked, every result against attention_ref.  Returns the raw outputs
    (out, lse, dqkv) for bit comparisons."""
    nkv = nh if nkv < 0 else nkv
    scale = 1.0 / math.sqrt(hd) if scale is None else scale
    case = f"B={B} T={T} nh={nh} nkv={nkv} hd={hd}{' interleaved' if interleaved else ''} {regime} scale={scale:.3g}"
    qkv = _operand(_qkv(B, T, nh, hd, nkv, interleaved, regime, scale, seed, batch_scale))
    out = _output(torch.empty(B * T, nh * hd, dtype=BF, device="cuda"))
    lse = _output(torch.empty(B * nh * T, dtype=F32, device="cuda"))
    C.attention_fwd(qkv, out.view, lse.view.view(B, nh, T), B, T, nh, hd, scale, interleaved, nkv)
    torch.cuda.synchronize()
    assert out.guards_intact() and lse.guards_intact(), f"{case}: the forward wrote outside out / lse"
    if regime == "do_eq_o":  # dO = O: dP - Δ cancels
        dout = _operand(out.view.clone())
    else:
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        dout = _operand((torch.randn(B * T, nh * hd, generator=g, device="cuda") * 0.5).to(BF))
    delta = _output(torch.empty(B * nh * T, dtype=F32, device="cuda"))
    dqkv = _output(torch.empty(qkv.shape, dtype=BF, device="cuda"))
    C.attention_bwd(qkv, out.view, dout, lse.view.view(B, nh, T), delta.view.view(B, nh, T), dqkv.view, B, T, nh, hd, scale, ws,
                    interleaved, nkv)
    torch.cuda.synchronize()
    assert delta.guards_intact() and dqkv.guards_intact(), f"{case}: the backward wrote outside delta / dqkv"
    r = ref.attention_ref(qkv, B, T, nh, hd, scale, interleaved, nkv, out=out.view, dout=dout)
    dq, dk, dv = ref.attention_unpack(dqkv.view, B, T, nh, hd, nkv=nkv, interleaved=interleaved)
    got = {"out": ref.attention_heads(out.view, B, T, nh, hd), "lse": lse.view.view(B, nh, T), "dq": dq, "dk": dk, "dv": dv}
    for name, val in got.items():
        _note(WORST, f"{family} {name}", ref.assert_attention_close(name, val, *r[name]), case)
    # delta = Σ_j dO·O' in fp32 from the bf16 out: a dot product, checked like an fp32 GEMM output
    O, dO = ref.attention_heads(out.view.double(), B, T, nh, hd), ref.attention_heads(dout.double(), B, T, nh, hd)
    ref.assert_gemm_close(delta.view.view(-1, 1), (O * dO).sum(-1).reshape(-1, 1), (O.abs() * dO.abs()).sum(-1).reshape(-1, 1))
    lse_ref, lse_b, lse_s, _ = r["lse"]
    err = (got["lse"].double() - lse_ref).abs()
    if bool((lse_s == 0).any()):
        _note(CALIB, "lse |err| / (1 + |lse|) where the score term is 0", float((err / lse_b)[lse_s == 0].max()), case)
    if bool((lse_s > 0).any()):
        _note(CALIB, "lse |err| / score term", float((err / lse_s)[lse_s > 0].max()), case)
    return out.view, lse.view, dqkv.view


# ----------------------------------------------------------------------------------------------- head sizes
@pytest.mark.parametrize("hd", [8, 16, 40, 48, 64, 72, 88, 104, 120, 128, 136, 152, 168, 192, 200, 216, 232, 256])
def test_head_sizes(C, hd):
    """Every K = 16 step count of mma_tiles_kk (hd % 16 = 8 meets zero-filled TMA columns), NP = 1..4 panels: the ragged dK/dV
    column split at NP = 3 and the split dQ at NP = 4."""
    _case(C, "head sizes", 2, 129, 2, hd, seed=hd)


def test_non_default_scale(C):
    _case(C, "head sizes", 2, 129, 2, 64, scale=0.3, seed=3)


# ----------------------------------------------------------------------------------------------- sequence tails
@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("hd", [64, 256])
@pytest.mark.parametrize("T", [1, 17, 63, 64, 65, 127, 128, 129, 1000, 2049])
def test_sequence_tails(C, T, hd, B):
    """The 64-row tiles past each sequence's tail hold the next batch's rows (each batch's v at its own scale)."""
    _case(C, "tails", B, T, 1, hd, seed=T + hd + B, batch_scale=True)


# ----------------------------------------------------------------------------------------------- grouped-query attention
@pytest.mark.parametrize("T", [33, 129, 1000])
@pytest.mark.parametrize("hd", [64, 128, 256])
@pytest.mark.parametrize("nh,nkv", [(4, 2), (8, 2), (16, 2), (4, 1)])
def test_grouped_query(C, nh, nkv, hd, T):
    """Groups of 2, 4 and 8, and one KV head; the last key block of every T takes the nblk == 1 && group > 1 prologue branch
    of the dK/dV kernel (at T <= 64 the only block)."""
    _case(C, "gqa", 2, T, nh, hd, nkv=nkv, seed=nh * 7 + nkv + hd + T, batch_scale=True)


# ----------------------------------------------------------------------------------------------- interleaved layout
@pytest.mark.parametrize("T", [129, 2049])
@pytest.mark.parametrize("hd", [64, 128, 256])
def test_interleaved_layout(C, hd, T):
    _case(C, "interleaved", 2, T, 2, hd, interleaved=True, seed=hd + T)


# ----------------------------------------------------------------------------------------------- score regimes
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("hd", [64, 128])
def test_score_regimes(C, hd, regime):
    _case(C, f"regime {regime}", 2, 1000, 2, hd, regime=regime, seed=hd + REGIMES.index(regime))


# ----------------------------------------------------------------------------------------------- shapes of the earlier sweeps
FOLDED = [  # (B, T, nh, hd, nkv): the multi-head, wide-head and grouped-query shapes the norm-relative sweeps ran
    (2, 512, 4, 48, 4), (1, 320, 2, 64, 2), (3, 128, 2, 32, 2), (1, 1000, 3, 64, 3), (2, 64, 1, 16, 1),
    (1, 320, 2, 80, 2), (2, 200, 2, 96, 2), (1, 1000, 2, 128, 2), (1, 130, 1, 136, 1), (1, 257, 2, 192, 2), (2, 64, 2, 256, 2),
    (1, 2049, 1, 256, 1),
] + [(B, T, (2 if hd == 64 else 1) * group, hd, 2 if hd == 64 else 1)
     for group in (1, 2, 4, 8) for hd in (64, 128) for B, T in ((2, 77), (1, 1000), (3, 64))]


@pytest.mark.parametrize("B,T,nh,hd,nkv", FOLDED)
def test_shapes_of_the_earlier_sweeps(C, B, T, nh, hd, nkv):
    _case(C, "earlier sweeps", B, T, nh, hd, nkv=nkv, seed=T + hd + nh)


# ----------------------------------------------------------------------------------------------- reproducibility
@pytest.mark.parametrize("B,T,nh,hd,nkv", [(2, 1000, 8, 128, 2), (2, 300, 2, 192, 2), (2, 300, 2, 256, 2)])
def test_backward_is_bit_reproducible_and_ignores_the_workspace(C, B, T, nh, hd, nkv):
    """Two runs agree bit for bit, and a NaN-filled ds_workspace changes nothing: the sm_90 kernels do not read it."""
    runs = [_case(C, "reproducibility", B, T, nh, hd, nkv=nkv, seed=9) for _ in range(2)]
    ws = torch.full((C.attention_ds_workspace_elems(B, T, nh),), float("nan"), dtype=BF, device="cuda")
    runs.append(_case(C, "reproducibility", B, T, nh, hd, nkv=nkv, seed=9, ws=ws))
    for other in runs[1:]:
        for x, y in zip(runs[0], other):
            assert torch.equal(x.view(torch.int16) if x.dtype == BF else x.view(torch.int32),
                               y.view(torch.int16) if y.dtype == BF else y.view(torch.int32))


# ----------------------------------------------------------------------------------------------- misaligned outputs
@pytest.mark.parametrize("where", ["column_offset", "odd_pitch"])
def test_misaligned_out_and_dqkv_are_refused(C, where):
    """The kernels read out with 16-byte loads and store 4-byte pairs into out / dqkv: a view that breaks 16-byte row alignment
    is refused on the host."""
    B, T, nh, hd = 1, 64, 2, 64
    h, W = nh * hd, 3 * nh * hd
    qkv = torch.randn(B * T, W, device="cuda").to(BF)
    lse = torch.empty(B, nh, T, dtype=F32, device="cuda")
    delta = torch.empty_like(lse)

    def bad(cols):
        if where == "column_offset":  # base 8 bytes past a 16-byte boundary
            return torch.zeros(B * T, cols + 8, dtype=BF, device="cuda")[:, 4:4 + cols]
        return torch.zeros(B * T, cols + 4, dtype=BF, device="cuda")[:, :cols]  # row pitch cols + 4

    good_out = torch.empty(B * T, h, dtype=BF, device="cuda")
    C.attention_fwd(qkv, good_out, lse, B, T, nh, hd, 0.125)
    dout = torch.randn(B * T, h, device="cuda").to(BF)
    with pytest.raises(RuntimeError, match="16-byte-aligned"):
        C.attention_fwd(qkv, bad(h), lse, B, T, nh, hd, 0.125)
    with pytest.raises(RuntimeError, match="16-byte-aligned"):
        C.attention_bwd(qkv, bad(h), dout, lse, delta, torch.empty_like(qkv), B, T, nh, hd, 0.125)
    with pytest.raises(RuntimeError, match="16-byte-aligned"):
        C.attention_bwd(qkv, good_out, dout, lse, delta, bad(W), B, T, nh, hd, 0.125)
    torch.cuda.synchronize()


# ----------------------------------------------------------------------------------------------- executor audit
class _Audit:
    """Wraps the extension's attention_fwd / attention_bwd: every call is checked against attention_ref on clones of its
    inputs (taken after a device synchronise), and its mode (direction, layout, panels per head) and count are recorded."""

    def __init__(self, C):
        self.fwd0, self.bwd0 = C.attention_fwd, C.attention_bwd
        self.modes, self.worst = {}, 0.0

    def _record(self, d, B, T, nh, hd, interleaved, nkv):
        layout = "interleaved" if interleaved else ("gqa" if 0 < nkv != nh else "mha")
        key = f"{d} {layout} NP={(hd + 63) // 64}"
        self.modes[key] = self.modes.get(key, 0) + 1

    def _check(self, r, got):
        for name, val in got.items():
            self.worst = max(self.worst, ref.assert_attention_close(name, val, *r[name]))

    def fwd(self, qkv, out, lse, B, T, nh, hd, scale, interleaved=False, nkv=-1):
        torch.cuda.synchronize()
        qc = qkv.clone()
        self.fwd0(qkv, out, lse, B, T, nh, hd, scale, interleaved, nkv)
        torch.cuda.synchronize()
        r = ref.attention_ref(qc, B, T, nh, hd, scale, interleaved, nkv)
        self._check(r, {"out": ref.attention_heads(out, B, T, nh, hd), "lse": lse.view(B, nh, T)})
        self._record("fwd", B, T, nh, hd, interleaved, nkv)

    def bwd(self, qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, scale, ds_workspace=None, interleaved=False, nkv=-1):
        torch.cuda.synchronize()
        qc, oc, dc = qkv.clone(), out.clone(), dout.clone()
        self.bwd0(qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, scale, ds_workspace, interleaved, nkv)
        torch.cuda.synchronize()
        r = ref.attention_ref(qc, B, T, nh, hd, scale, interleaved, nkv, out=oc, dout=dc)
        dq, dk, dv = ref.attention_unpack(dqkv, B, T, nh, hd, nkv=nh if nkv < 0 else nkv, interleaved=interleaved)
        self._check(r, {"dq": dq, "dk": dk, "dv": dv})
        self._record("bwd", B, T, nh, hd, interleaved, nkv)

    def install(self, monkeypatch, C):
        monkeypatch.setattr(C, "attention_fwd", self.fwd)
        monkeypatch.setattr(C, "attention_bwd", self.bwd)


def _info():
    from relora_b200.parallel.dist import DistInfo

    return DistInfo(0, 0, 1, torch.device("cuda", 0), "nccl")


def _llama_cfg(hidden, nh, nkv):
    from relora_b200.models import SimpleConfig

    return SimpleConfig(model_type="llama", vocab_size=1024, hidden_size=hidden, intermediate_size=512, num_hidden_layers=2,
                        num_attention_heads=nh, num_key_value_heads=nkv, rope_theta=10000.0, rms_norm_eps=1e-6, pad_token_id=-1,
                        max_position_embeddings=256)


def _relora_llama(hidden, nh, nkv):
    from relora_b200.models import LlamaForCausalLM
    from relora_b200.relora import ReLoRaModel

    torch.manual_seed(0)
    w = ReLoRaModel(LlamaForCausalLM(_llama_cfg(hidden, nh, nkv)), r=128, lora_alpha=32, lora_dropout=0.1,
                    target_modules=["attn", "mlp"], init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    return w.cuda().to(BF)


def _pythia():
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.relora import ReLoRaModel

    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=1024, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                       intermediate_size=1024, rotary_pct=0.25, max_position_embeddings=128, layer_norm_eps=1e-5,
                       use_parallel_residual=True, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    torch.manual_seed(0)
    w = ReLoRaModel(GPTNeoXForCausalLM(cfg), r=128, lora_alpha=32, lora_dropout=0.1, target_modules=["attn", "attention", "mlp"],
                    init_lora_a="kaiming")
    with torch.no_grad():
        for mod in w.relora_modules():
            torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
            torch.nn.init.normal_(mod.bias, std=0.02)
    return w.cuda().to(BF).train()


_AUDIT = {  # configuration -> the call forms of one micro-step and one eval_loss (module path: one forward / backward); a path
    # that starts issuing another form shows up here
    "llama_mha_auto": {"fwd mha NP=1", "bwd mha NP=1"},
    "llama_gqa": {"fwd gqa NP=1", "bwd gqa NP=1"},
    "llama_hd128_native": {"fwd mha NP=2", "bwd mha NP=2"},
    "pythia_parallel": {"fwd interleaved NP=1", "bwd interleaved NP=1"},
    "module_path": {"fwd mha NP=1", "bwd mha NP=1"},
}


@pytest.mark.parametrize("config", list(_AUDIT))
def test_executor_attention_matches_the_reference(C, config, monkeypatch):
    """Every attention call of one training micro-step and one evaluation (CUDA graphs off, 3 x 97 tokens), or of one module-path
    forward / backward, checked against attention_ref; the modes seen and their counts must be the expected ones."""
    from relora_b200.ops import fused

    dev = torch.device("cuda", 0)
    ids = torch.randint(0, 1024, (3, 97), device=dev)
    audit = _Audit(C)
    if config == "module_path":
        from relora_b200.models import LlamaForCausalLM

        monkeypatch.setenv("RELORA_B200_ATTENTION", "native")
        torch.manual_seed(0)
        m = LlamaForCausalLM(_llama_cfg(256, 4, 4)).to("cuda", BF).train()
        audit.install(monkeypatch, C)
        loss = m(input_ids=ids, labels=ids).loss
        loss.backward()
        assert torch.isfinite(loss)
    else:
        monkeypatch.delenv("RELORA_B200_ATTENTION", raising=False)
        if config == "pythia_parallel":
            from relora_b200.engine.fused_pythia import FusedPythiaStepper

            st = FusedPythiaStepper(_pythia(), _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False)
        else:
            from relora_b200.engine.fused_llama import FusedLlamaStepper

            hidden, nh, nkv, attention = {"llama_mha_auto": (256, 4, 4, "auto"), "llama_gqa": (256, 4, 2, "auto"),
                                          "llama_hd128_native": (256, 2, 2, "native")}[config]
            st = FusedLlamaStepper(_relora_llama(hidden, nh, nkv), _info(), lr=1e-3, grad_accumulation=1, cuda_graphs=False,
                                   attention=attention)
        assert st.native_attn
        fused.seed_state.set(dev, 4321)
        audit.install(monkeypatch, C)
        loss = st.micro_step(ids)
        ev = st.eval_loss(ids)
        assert torch.isfinite(loss) and torch.isfinite(ev)
    calls = sum(audit.modes.values())
    print(f"[attention modes] audit {config}: {calls} calls, worst ratio {audit.worst:.3g}, modes {dict(sorted(audit.modes.items()))}")
    _note(WORST, "audit", audit.worst, config)
    assert set(audit.modes) == _AUDIT[config]
