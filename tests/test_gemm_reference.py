"""The fp64 reference of the wgmma GEMM contract (ops/reference.py: gemm_ref, lora_dx_ref) and its comparator
assert_gemm_close, on the CPU: the reference agrees with the per-group composition the executors' docstrings state, and
the tolerance rejects a single structural error at the shapes the GPU sweep (test_gemm_modes_gpu.py) uses."""
import pytest
import torch

from gemm_forms import FORMS, lora_group_call, lora_group_composition, lora_group_shapes
from relora_b200.ops import reference as ref

BF = torch.bfloat16
F64 = torch.float64
M_TOK, K_H, R = 291, 256, 128  # ragged token count, hidden size, LoRA rank of the GPU sweep


def _tensors(shapes, seed=0):
    g = torch.Generator().manual_seed(seed)
    T = {}
    for name, (shape, dt) in shapes.items():
        scale = 0.05 if name in ("A", "W", "B") else (0.1 if name == "bias" else 1.0)
        T[name] = (torch.randn(*shape, generator=g) * scale).to(dt)
    return T


@pytest.mark.parametrize("G,Ng", [(1, 256), (2, 384), (3, 256)])
@pytest.mark.parametrize("drop", [False, True])
@pytest.mark.parametrize("form", FORMS)
def test_gemm_ref_matches_the_per_group_composition(form, G, Ng, drop):
    dims = dict(G=G, K=K_H, Ng=Ng, r=R)
    T = _tensors(lora_group_shapes(M=M_TOK, drop=drop, **dims), seed=G * 10 + len(form))
    a1, b1, out, kw = lora_group_call(form, T, M=M_TOK, s=0.25, drop=drop, **dims)
    got, bound = ref.gemm_ref(a1, b1, out, **kw)
    want = lora_group_composition(form, T, s=0.25, drop=drop, **dims)
    assert got.shape == want.shape
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    assert bool((bound >= got.abs() - 1e-9).all())


def test_gemm_ref_operand_forms_fp8_alpha_dev_and_accumulate():
    g = torch.Generator().manual_seed(1)
    M, N, K = 33, 40, 72
    a, b = torch.randn(M, K, generator=g).to(BF), torch.randn(N, K, generator=g).to(BF)
    want = a.double() @ b.double().t()
    for a_mn in (False, True):
        for b_mn in (False, True):
            got, _ = ref.gemm_ref(a.t().contiguous() if a_mn else a, b.t().contiguous() if b_mn else b, M=M, N=N, K1=K,
                                  a1_mn=a_mn, b1_mn=b_mn)
            torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    # alpha x alpha_dev, then bf16 accumulate onto the previous output
    prev = torch.randn(M, N, generator=g).to(BF)
    got, bound = ref.gemm_ref(a, b, prev, alpha=0.5, alpha_dev=torch.tensor([3.0]), accumulate=True)
    torch.testing.assert_close(got, 1.5 * want + prev.double(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(bound, 1.5 * (a.double().abs() @ b.double().abs().t()) + prev.double().abs(), rtol=1e-12, atol=1e-12)
    # fp8: bytes decoded as E4M3, A1 as E5M2 with fp8=2
    a8, b8 = (a.float() * 4).to(torch.float8_e5m2), b.float().to(torch.float8_e4m3fn)
    got, _ = ref.gemm_ref(a8.view(torch.uint8), b8.view(torch.uint8), fp8=2)
    torch.testing.assert_close(got, a8.double() @ b8.double().t(), rtol=1e-12, atol=1e-12)
    a8 = a.float().to(torch.float8_e4m3fn)
    got, _ = ref.gemm_ref(a8.view(torch.uint8), b8.view(torch.uint8), fp8=1)
    torch.testing.assert_close(got, a8.double() @ b8.double().t(), rtol=1e-12, atol=1e-12)


def test_gemm_ref_rejects_what_the_kernel_does_not_define():
    a, b = torch.zeros(8, 64, dtype=BF), torch.zeros(16, 64, dtype=BF)
    with pytest.raises(ValueError):
        ref.gemm_ref(a, b, torch.zeros(8, 16), bias=torch.zeros(16, dtype=BF))
    with pytest.raises(ValueError):
        ref.gemm_ref(a, b, torch.zeros(8, 16), residual=torch.zeros(8, 16, dtype=BF))
    with pytest.raises(IndexError):  # the second group's K window would leave A1
        ref.gemm_ref(a, torch.zeros(16, 64, dtype=BF), M=8, N=16, K1=64, n_per_group=8, a1_group_kofs=64,
                     b1_group_kofs=0)


def test_lora_dx_ref_matches_masked_sum():
    g = torch.Generator().manual_seed(2)
    M, N, G, r, Kb, p, seed, keys = 37, 64, 2, 64, 96, 0.25, 1234567, [11, 22]
    dy, w = torch.randn(M, Kb, generator=g).to(BF), torch.randn(Kb, N, generator=g).to(BF)
    du, a = torch.randn(M, G * r, generator=g).to(BF), torch.randn(G * r, N, generator=g).to(BF)
    want = dy.double() @ w.double()
    for i in range(G):
        keep = ref.dropout_keep_mask(ref.mix_seed(seed, keys[i]), M, N, p)
        want += keep * (du[:, i * r:(i + 1) * r].double() @ a[i * r:(i + 1) * r].double()) / (1 - p)
    got, _ = ref.lora_dx_ref(dy, w, du, a, torch.tensor([seed], dtype=torch.int32), keys, p)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    base = (dy.double() @ w.double()).to(BF)
    got, _ = ref.lora_dx_ref(None, None, du, a, seed, keys, p, base=base)
    torch.testing.assert_close(got, want - dy.double() @ w.double() + base.double(), rtol=1e-12, atol=1e-12)


def test_assert_gemm_close_reports_the_worst_element_and_fails_on_nan():
    r = torch.ones(4, 5, dtype=F64)
    assert ref.assert_gemm_close(r.to(BF), r, r) == 0.0
    out = r.clone().float()
    out[2, 3] = 1.5
    with pytest.raises(AssertionError, match=r"row 2, col 3"):
        ref.assert_gemm_close(out, r, r)
    out[2, 3] = float("nan")
    with pytest.raises(AssertionError, match="1 of 20"):
        ref.assert_gemm_close(out, r, r)


# ---------------------------------------------------------------------------------------------- sensitivity
def _mutation(name):
    """(output of a kernel with one structural error, exact reference, bound, fp8) at a GPU-sweep shape."""
    if name in ("kblock_dropped", "window_shifted", "mgroup_offset"):
        dims = dict(G=3, K=K_H, Ng=256, r=R)
        T = _tensors(lora_group_shapes(M=M_TOK, drop=True, **dims), seed=3)
        form = "dA" if name == "mgroup_offset" else "u"
        a1, b1, out, kw = lora_group_call(form, T, M=M_TOK, s=0.25, drop=True, **dims)
        want, bound = ref.gemm_ref(a1, b1, out, **kw)
        if name == "mgroup_offset":  # M-tile 1 (rows 128..255, m-group 1) reads the B1 rows of m-group 0
            alt, _ = ref.gemm_ref(a1, b1, out, **dict(kw, b1_mn_ofs_per_mgroup=0))
            bad = want.clone()
            bad[128:256] = alt[128:256]
            return bad.float(), want, bound
        xd = T["xd"].clone()
        if name == "kblock_dropped":  # group 1 skips its second k-block
            xd[:, K_H + 64:K_H + 128] = 0
        else:  # group 1 reads its K window 64 columns late
            xd[:, K_H:2 * K_H] = T["xd"][:, K_H + 64:2 * K_H + 64]
        bad, _ = ref.gemm_ref(xd, b1, out, **kw)
        return bad.to(BF), want, bound
    if name in ("bias_column", "residual_row"):
        dims = dict(G=3, K=K_H, Ng=256, r=R)
        T = _tensors(lora_group_shapes(M=M_TOK, drop=False, **dims), seed=4)
        a1, b1, out, kw = lora_group_call("y", T, M=M_TOK, s=0.25, drop=False, **dims)
        want, bound = ref.gemm_ref(a1, b1, out, **kw)
        bad = want.clone()
        if name == "bias_column":
            bad[:, 517] -= T["bias"][517].double()
        else:
            bad[200] -= T["res"][200].double()
        return bad.to(BF), want, bound
    if name == "odd_n_last_column":
        g = torch.Generator().manual_seed(5)
        a, b = torch.randn(129, 72, generator=g).to(BF), (torch.randn(1001, 72, generator=g) * 0.05).to(BF)
        want, bound = ref.gemm_ref(a, b)
        bad = want.clone()
        bad[:, -1] = 0
        return bad.to(BF), want, bound
    if name == "lora_dx_mask_swapped":
        g = torch.Generator().manual_seed(6)
        M, G, Ng, N, p, keys = M_TOK, 3, 256, 256, 0.1, [11, 22, 33]
        dy, w = torch.randn(M, G * Ng, generator=g).to(BF), (torch.randn(G * Ng, N, generator=g) * 0.05).to(BF)
        du, a = torch.randn(M, G * R, generator=g).to(BF), (torch.randn(G * R, N, generator=g) * 0.05).to(BF)
        want, bound = ref.lora_dx_ref(dy, w, du, a, 1234567, keys, p)
        bad, _ = ref.lora_dx_ref(dy, w, du, a, 1234567, [22, 11, 33], p)
        return bad.to(BF), want, bound
    raise ValueError(name)


@pytest.mark.parametrize("name", ["kblock_dropped", "window_shifted", "bias_column", "residual_row", "mgroup_offset",
                                  "odd_n_last_column", "lora_dx_mask_swapped"])
def test_assert_gemm_close_rejects_one_structural_error(name):
    bad, want, bound = _mutation(name)
    assert ref.assert_gemm_close(want.to(bad.dtype), want, bound) <= 1.0  # the exact result, rounded, passes
    with pytest.raises(AssertionError):
        ref.assert_gemm_close(bad, want, bound)
    with pytest.raises(AssertionError):  # ... also with the fp8 accumulation tolerance
        ref.assert_gemm_close(bad, want, bound, fp8=True)
