"""CTA pairs of the wgmma GEMM and of the LoRA input-gradient kernel, and the latter's TMA-store epilogue.

A pair computes two M tiles of one N tile from one B tile that each CTA loads half of.  Per-tile k order and epilogue
arithmetic are those of a single CTA, so a paired call must give the bits of the unpaired call for every form the executors
issue; split-K sums through fp32 atomics in no fixed order and is checked against the fp64 reference instead.  The
operands sit inside NaN-guarded buffers and the outputs inside sentinel-guarded ones (guarded_buffers.py)."""
import pytest
import torch

from gemm_forms import FORMS, lora_group_call, lora_group_shapes
from guarded_buffers import Guarded
from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
R = 128
SENTINEL = 1234.0


@pytest.fixture(scope="module")
def F():
    from relora_b200.ops import fused

    fused._C()
    return fused


def _operand(t):
    return Guarded(t, 0x7F if t.dtype == torch.uint8 else float("nan"), pitch_multiple=16).view


def _rand(*shape, scale=1.0, dtype=BF):
    return (torch.randn(*shape, device="cuda") * scale).to(dtype)


def _gemm(F, a1, b1, out_t, pair, **kw):
    """one call on guarded operands; returns the output (guards checked) and the output's value before the call"""
    acc = bool(kw.get("accumulate", False))
    ops = {k: (_operand(v) if torch.is_tensor(v) and k != "alpha_dev" else v) for k, v in kw.items()}
    o = Guarded(out_t, SENTINEL, interior=None if acc else torch.full_like(out_t, float("nan")))
    prev = o.view.clone()
    A1, B1 = _operand(a1), _operand(b1)
    F.gemm(A1, B1, o.view, pair=pair, **ops)
    torch.cuda.synchronize()
    assert o.guards_intact(), "the output guard region was written"
    return o.view.clone(), (A1, B1, prev, ops)


def _same_bits(F, a1, b1, out_t, **kw):
    got0, _ = _gemm(F, a1, b1, out_t, 0, **kw)
    got1, (A1, B1, prev, ops) = _gemm(F, a1, b1, out_t, 1, **kw)
    assert not torch.isnan(got1).any()
    assert torch.equal(got0, got1), f"paired differs from unpaired in {int((got0 != got1).sum())} elements"
    want, bound = ref.gemm_ref(A1, B1, prev, **ops)
    ref.assert_gemm_close(got1, want, bound, fp8=bool(kw.get("fp8", 0)))


def _group_tensors(G, K, Ng, M, drop, seed):
    torch.manual_seed(seed)
    T = {}
    for name, (shape, dt) in lora_group_shapes(G=G, K=K, Ng=Ng, M=M, r=R, drop=drop).items():
        T[name] = _rand(*shape, scale=0.05 if name in ("A", "W", "B") else (0.1 if name == "bias" else 1.0), dtype=dt)
    return T


# M 12416 and 328: an odd number of M tiles, so the last pair's second tile lies past M (328 also ragged inside a tile).
# The dA / dB forms run with M = G·r or G·Ng and M groups of r or Ng rows: groups of 256 rows pair, groups of 128 do not.
@pytest.mark.parametrize("M", [328, 12416])
@pytest.mark.parametrize("G,Ng,drop", [(1, 256, False), (2, 384, True), (3, 256, True)])
@pytest.mark.parametrize("form", FORMS)
def test_forms_paired_equal_unpaired(F, form, G, Ng, drop, M):
    if M > 1000 and form in ("dA", "dB") and G != 3:
        pytest.skip("the long-reduction weight gradients are covered at G = 3")
    T = _group_tensors(G, 256, Ng, M, drop, seed=G * 7 + M)
    a1, b1, out, kw = lora_group_call(form, T, G=G, K=256, Ng=Ng, M=M, r=R, s=0.25, drop=drop, split_k=1)
    _same_bits(F, a1, b1, out, **kw)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(328, 128, 200), (12416, 128, 768), (1000, 1001, 72)])
def test_plain_majors(F, M, N, K, a_mn, b_mn):
    """N 128 (one N tile: u_o / u_d / du_* sites), both majors of both operands, ragged N and K"""
    torch.manual_seed(M + N + K)
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    _same_bits(F, a.t().contiguous() if a_mn else a, b.t().contiguous() if b_mn else b,
               torch.empty(M, N, dtype=BF, device="cuda"), M=M, N=N, K1=K, a1_mn=a_mn, b1_mn=b_mn)


@pytest.mark.parametrize("Ng", [256, 320])
def test_grouped_ragged_windows_bias_residual(F, Ng):
    """two groups with per-group K windows on A1 and A2; Ng 320 leaves each group a ragged last N tile"""
    M, K, G = 328, 256, 2
    torch.manual_seed(Ng)
    N = G * Ng
    _same_bits(F, _rand(M, G * K), _rand(N, K, scale=0.05), torch.empty(M, N, dtype=BF, device="cuda"), M=M, N=N, K1=K,
               n_per_group=Ng, a1_group_kofs=K, a2=_rand(M, G * R), b2=_rand(N, R, scale=0.05), K2=R, a2_group_kofs=R,
               bias=_rand(N, scale=0.1), residual=_rand(M, N), alpha=0.5)


@pytest.mark.parametrize("odt", [BF, F32])
def test_accumulate(F, odt):
    M, N, K = 328, 384, 320
    torch.manual_seed(5)
    _same_bits(F, _rand(M, K), _rand(N, K, scale=0.05), _rand(M, N).to(odt), M=M, N=N, K1=K, accumulate=True, alpha=2.0)


def _quant(x, dtype):
    s = float(x.float().abs().max()) / torch.finfo(dtype).max
    return (x.float() / s).to(dtype).view(torch.uint8), s


@pytest.mark.parametrize("fp8", [1, 2])
def test_fp8_segment(F, fp8):
    """E4M3 (fp8=1, with the bf16 LoRA segment) and E5M2 x E4M3 (fp8=2) K-major segment 1"""
    M, N, K = 328, 768, 320
    torch.manual_seed(fp8)
    (x8, sx), (w8, sw) = _quant(_rand(M, K), torch.float8_e4m3fn if fp8 == 1 else torch.float8_e5m2), \
        _quant(_rand(N, K, scale=0.05), torch.float8_e4m3fn)
    kw = dict(M=M, N=N, K1=K, fp8=fp8, alpha_dev=torch.tensor([sx * sw], dtype=F32, device="cuda"))
    if fp8 == 1:
        kw.update(a2=(_rand(M, R).float() / (sx * sw)).to(BF), b2=_rand(N, R, scale=0.05), K2=R)
    _same_bits(F, x8, w8, torch.empty(M, N, dtype=BF, device="cuda"), **kw)


@pytest.mark.parametrize("split_k", [0, 7])
@pytest.mark.parametrize("form", ["dA", "dB"])
def test_split_k_paired(F, form, split_k):
    """split-K with pair=1 (fp32 atomics: checked against the fp64 reference, not bit for bit)"""
    G, Ng, M = 1, 512, 4098
    T = _group_tensors(G, 512, Ng, M, False, seed=31)
    a1, b1, out, kw = lora_group_call(form, T, G=G, K=512, Ng=Ng, M=M, r=R, s=0.25, drop=False, split_k=split_k)
    got, (A1, B1, prev, ops) = _gemm(F, a1, b1, out, 1, **kw)
    want, bound = ref.gemm_ref(A1, B1, prev, **ops)
    ref.assert_gemm_close(got, want, bound)


# ----------------------------------------------------------------------------------------------- lora_dx
def _lora_dx(C, T, N, with_base, pair):
    o = Guarded(torch.empty(T["M"], N, dtype=BF, device="cuda"), SENTINEL, interior=torch.full((T["M"], N), float("nan"),
                                                                                               dtype=BF, device="cuda"))
    A = T["A"][:, :N]
    if with_base:
        C.lora_dx(None, None, T["du"], A, o.view, T["seed"], T["keys"], 0.1, T["base"][:, :N], pair=pair)
    else:
        C.lora_dx(T["dy"], T["W"][:, :N], T["du"], A, o.view, T["seed"], T["keys"], 0.1, pair=pair)
    torch.cuda.synchronize()
    assert o.guards_intact(), "the output guard region was written"
    return o.view.clone()


@pytest.mark.parametrize("with_base", [False, True])
@pytest.mark.parametrize("G,M", [(1, 328), (3, 12416), (2, 129)])
def test_lora_dx_pairs_and_tma_store(F, G, M, with_base):
    """N 1000 (a multiple of 8, not of 128) stores through TMA; N 1002 keeps the register epilogue, whose first 1000 columns
    are the same product (each column depends only on its own operand columns and the (row, col) dropout hash).  Paired and
    unpaired, both forms must give the same bits, with dropout p = 0.1."""
    C = F._C()
    torch.manual_seed(G * 100 + M)
    Ng, Nmax = 256, 1002
    T = {"M": M, "keys": [11, 22, 33][:G], "seed": torch.tensor([1234567], dtype=torch.int32, device="cuda"),
         "dy": _operand(_rand(M, G * Ng)), "W": _operand(_rand(G * Ng, Nmax, scale=0.05)), "du": _operand(_rand(M, G * R)),
         "A": _operand(_rand(G * R, Nmax, scale=0.05)), "base": _operand(_rand(M, Nmax))}
    tma0, tma1 = _lora_dx(C, T, 1000, with_base, 0), _lora_dx(C, T, 1000, with_base, 1)
    reg0, reg1 = _lora_dx(C, T, 1002, with_base, 0), _lora_dx(C, T, 1002, with_base, 1)
    assert not torch.isnan(tma1).any() and not torch.isnan(reg1).any()
    assert torch.equal(tma0, tma1), "paired TMA-store output differs from unpaired"
    assert torch.equal(reg0, reg1), "paired register-epilogue output differs from unpaired"
    assert torch.equal(tma0, reg0[:, :1000]), "TMA-store epilogue differs from the register epilogue"
    want, bound = ref.lora_dx_ref(None if with_base else T["dy"], None if with_base else T["W"][:, :1000], T["du"],
                                  T["A"][:, :1000], T["seed"], T["keys"], 0.1, base=T["base"][:, :1000] if with_base else None)
    ref.assert_gemm_close(tma1, want, bound)
