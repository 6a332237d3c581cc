"""The fp64 references of the row-wise kernels (ops/reference.py, row-wise section) and their comparators on the CPU: each
reference agrees with fp64 autograd or an independent plain expression at the shapes the GPU sweep (test_rowwise_modes_gpu.py)
uses, a correctly rounded result passes, and the comparators reject each structural defect a kernel could have."""
import math

import pytest
import torch
import torch.nn.functional as F

from relora_b200.ops import reference as ref

BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rms_inputs(M, H, seed):
    g = _g(seed)
    x = (torch.randn(M, H, generator=g) * 2.0 + 0.1).to(BF)
    w = (1.0 + 0.3 * torch.randn(H, generator=g)).to(BF)
    dy = torch.randn(M, H, generator=g).to(BF)
    rstd = torch.rsqrt(x.float().pow(2).mean(-1) + 1e-5)
    return x, w, dy, rstd


def _fails(fn, *args):
    with pytest.raises(AssertionError):
        fn(*args)


# ----------------------------------------------------------------------------------------------- agreement with autograd
@pytest.mark.parametrize("M,H", [(7, 8), (9, 264), (33, 2056)])
def test_rmsnorm_reference_agrees_with_the_module_definition_and_autograd(M, H):
    x, w, dy, rstd = _rms_inputs(M, H, M + H)
    r = ref.rmsnorm_fwd_ref(x, w, 1e-5, rstd)
    assert torch.equal(r["y"], ref.rmsnorm(x, w, 1e-5))  # the module path's rounding order, bit for bit
    r64, b = r["rstd"]
    assert torch.allclose(r64, 1.0 / torch.sqrt(x.double().pow(2).mean(-1) + 1e-5), rtol=1e-12) and bool((b > 0).all())
    ref.assert_rowwise_close("rstd", rstd, r64, b)
    # dx: autograd of w·x·rstd(x) with the fp64 rstd; the reference reads the stored fp32 rstd, so they agree to ~2^-24
    X = x.double().requires_grad_()
    (w.double() * X * torch.rsqrt(X.pow(2).mean(-1, keepdim=True) + 1e-5)).backward(dy.double())
    add = torch.randn(M, H, generator=_g(1)).to(BF)
    rb = ref.rmsnorm_bwd_ref(dy, x, w, rstd, add, torch.ones(H))
    assert torch.allclose(rb["dx"][0], X.grad + add.double(), rtol=1e-5, atol=1e-5)
    xhb = (x.float() * rstd[:, None]).to(BF).double()
    assert torch.allclose(rb["dw"][0], 1.0 + (dy.double() * xhb).sum(0), rtol=1e-12)


@pytest.mark.parametrize("M,H,offset", [(9, 136, 0.0), (40, 1032, 64.0)])
def test_layernorm_reference_agrees_with_autograd(M, H, offset):
    g = _g(H)
    x = (torch.randn(M, H, generator=g) + offset).to(BF)
    w1, w2 = [(1.0 + 0.3 * torch.randn(H, generator=g)).to(BF) for _ in range(2)]
    b1 = (0.2 * torch.randn(H, generator=g)).to(BF)
    dy1, dy2, dres = [torch.randn(M, H, generator=g).to(BF) for _ in range(3)]
    X = x.double()
    mu, var = X.mean(-1), X.var(-1, unbiased=False)
    r = ref.layernorm_fwd_ref(x, 1e-5, mu.float(), torch.rsqrt(var + 1e-5).float(), [(w1, b1), (w2, None)])
    assert torch.allclose(r["mean"][0], mu, rtol=1e-12) and torch.allclose(r["rstd"][0], 1 / torch.sqrt(var + 1e-5), rtol=1e-6)
    assert torch.allclose(r["y0"][0], F.layer_norm(X, (H,), w1.double(), b1.double(), 1e-5), rtol=1e-5, atol=1e-5)
    assert torch.allclose(r["y1"][0], F.layer_norm(X, (H,), w2.double(), None, 1e-5), rtol=1e-5, atol=1e-5)
    Xg = X.clone().requires_grad_()
    W1, B1, W2 = (t.double().requires_grad_() for t in (w1, b1, w2))
    (F.layer_norm(Xg, (H,), W1, B1, 1e-5) * dy1.double() + F.layer_norm(Xg, (H,), W2, None, 1e-5) * dy2.double()).sum().backward()
    zeros = torch.zeros(H)
    rb = ref.layernorm_bwd_ref(x, mu.float(), torch.rsqrt(var + 1e-5).float(), [(dy1, w1, zeros, zeros), (dy2, w2, zeros, None)],
                               dres, (zeros, torch.ones(H)))
    assert torch.allclose(rb["dx"][0], Xg.grad + dres.double(), rtol=1e-4, atol=1e-4)
    assert torch.allclose(rb["dw0"][0], W1.grad, rtol=1e-4, atol=1e-4) and torch.allclose(rb["db0"][0], B1.grad, rtol=1e-9)
    assert torch.allclose(rb["dw1"][0], W2.grad, rtol=1e-4, atol=1e-4) and "db1" not in rb
    assert torch.allclose(rb["dres_sum0"][0] + 1.0, rb["dres_sum1"][0], rtol=1e-12)


@pytest.mark.parametrize("V", [8, 1001, 1007, 32100])
def test_cross_entropy_reference_agrees_with_autograd(V):
    M = 11
    g = _g(V)
    x = (torch.randn(M, V, generator=g) * 2.0).to(BF)
    lab = torch.randint(0, V, (M,), generator=g)
    lab[1], lab[3] = V - 1, -100
    X = x.double().requires_grad_()
    loss = F.cross_entropy(X, lab, ignore_index=-100, reduction="sum")
    loss.backward()
    r = ref.cross_entropy_ref(x, lab, V, 0.37, -100, torch.tensor([2.5]), torch.tensor([3.0]))
    assert torch.allclose(r["grad"][0], 0.37 * X.grad, rtol=1e-12, atol=1e-15)
    assert torch.allclose(r["loss_sum"][0], 2.5 + loss.detach().reshape(1), rtol=1e-12)
    assert float(r["count"]) == 3.0 + (M - 1)
    assert torch.equal(r["grad"][0][3], torch.zeros(V, dtype=F64))


@pytest.mark.parametrize("hd,rot,backward", [(64, 64, False), (64, 16, True), (128, 8, False)])
def test_rope_references_agree_with_the_half_rotation(hd, rot, backward):
    T, nh, nkv, pos0 = 9, 2, 1, 3
    cos, sin = ref.rope_tables(rot, T + pos0)
    cos, sin = cos.to(BF), sin.to(BF)
    x = torch.randn(2 * T, (nh + 2 * nkv) * hd, generator=_g(hd + rot)).to(BF)
    mask, r, b = ref.rope_inplace_ref(x, T, nh + nkv, hd, rot, cos, sin, backward, pos0)
    s = (-1.0 if backward else 1.0) * sin.double()
    heads = x.double().view(2, T, nh + 2 * nkv, hd)
    rotd = ref.rope_apply(heads[..., :rot].transpose(1, 2), cos.double()[pos0:pos0 + T], s[pos0:pos0 + T]).transpose(1, 2)
    want = heads.clone()
    want[:, :, :nh + nkv, :rot] = rotd[:, :, :nh + nkv]
    assert torch.allclose(r, want.reshape_as(r), rtol=1e-12)
    assert int(mask.sum()) == 2 * T * (nh + nkv) * rot
    # rope_pack_bwd of [B, heads, T, hd] views is the backward rotation of the packed buffer
    q, k, v = ref.attention_unpack(x, 2, T, nh, hd, nkv=nkv)
    ex, r2, _ = ref.rope_pack_bwd_ref(q, k, v, rot, cos, sin, pos0)
    _, r3, _ = ref.rope_inplace_ref(x, T, nh + nkv, hd, rot, cos, sin, True, pos0)
    assert torch.equal(r2, r3) and int((~ex).sum()) == int(mask.sum())
    # neox layout: q and k of each head rotated, v untouched
    xn = torch.randn(2 * T, nh * 3 * hd, generator=_g(1)).to(BF)
    mn, rn, _ = ref.neox_rope_ref(xn, T, nh, hd, rot, cos.float(), sin.float(), pos0, backward)
    assert int(mn.sum()) == 2 * T * nh * 2 * rot and torch.equal(rn[~mn], xn.double()[~mn])


def test_activation_references_agree_with_autograd():
    g = _g(5)
    z = torch.cat([torch.linspace(-90, 90, 64), torch.randn(136, generator=g) * 3]).view(4, 50).to(BF)
    u = torch.randn(4, 50, generator=g).to(BF)
    dh = torch.randn(4, 50, generator=g).to(BF)
    Z, U = z.double().requires_grad_(), u.double().requires_grad_()
    (F.silu(Z) * U).backward(dh.double())
    gu = torch.cat([z, u], 1)
    h, _ = ref.swiglu_fwd_ref(gu, 50)
    assert torch.allclose(h, F.silu(z.double()) * u.double(), rtol=1e-12, atol=1e-300)
    rb = ref.swiglu_bwd_ref(dh, gu, 50)
    assert torch.allclose(rb["dg"][0], Z.grad, rtol=1e-10, atol=1e-300) and torch.allclose(rb["du"][0], U.grad, rtol=1e-10)
    for approx in (False, True):
        Zg = z.double().requires_grad_()
        a = F.gelu(Zg, approximate="tanh" if approx else "none")
        a.backward(dh.double())
        # 1 + erf(z/√2) and 1 + tanh cancel for z << 0, where autograd's own fp64 value is only absolutely accurate
        assert torch.allclose(ref.gelu_fwd_ref(z, approx)[0], a.detach(), rtol=1e-12, atol=1e-13)
        assert torch.allclose(ref.gelu_bwd_ref(dh, z, approx)[0], Zg.grad, rtol=1e-10, atol=1e-13)


def test_adamw_reference_agrees_with_the_fp32_step():
    g = _g(7)
    n = 1000
    p, grad = torch.randn(n, generator=g).to(BF), torch.randn(n, generator=g) * 0.01
    m, v = torch.randn(n, generator=g) * 0.01, torch.rand(n, generator=g) * 1e-4
    for step in (1, 10000):
        r = ref.adamw_ref(p, grad, m, v, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=0.1, step=step, grad_scale=0.5)
        P, M_, V_ = p.clone(), m.clone(), v.clone()
        f32 = lambda a: float(torch.tensor(a, dtype=F32))  # noqa: E731  the kernel's hyperparameters: 1 - 0.999f is not 0.001
        ref.adamw_step(P, grad, M_, V_, step=step, lr=f32(1e-3), beta1=f32(0.9), beta2=f32(0.999), eps=f32(1e-8),
                       weight_decay=f32(0.1), grad_scale=0.5)
        ref.assert_rowwise_close("p", P, *r["p"])
        ref.assert_rowwise_close("m", M_, *r["m"])
        ref.assert_rowwise_close("v", V_, *r["v"])


def test_exact_references():
    g = _g(9)
    # embedding_bwd_sorted: a plain position-ordered fp32 loop
    ids = torch.randint(0, 5, (40,), generator=g)
    dout = torch.randn(40, 16, generator=g).to(BF)
    before = torch.randn(5, 16, generator=g)
    srt = torch.sort(ids, stable=True)
    got = ref.embedding_bwd_sorted_exact(srt.values, srt.indices, dout, before, 2)
    want = before.clone()
    for i in range(5):
        if i == 2:
            continue
        acc = torch.zeros(16)
        for pos in range(40):
            if int(ids[pos]) == i:
                acc = acc + dout[pos].float()
        want[i] = want[i] + acc
    assert torch.equal(got, want)
    # dropout copy: the mask of dropout_keep_mask times fp32 1/(1-p)
    y = torch.randn(6, 24, generator=g).to(BF)
    keep = ref.dropout_keep_mask(ref.mix_seed(77, 3), 6, 24, 0.25)
    assert torch.equal(ref.dropout_copy_exact(y, 77, 3, 0.25), (y.float() * keep * (1 / 0.75)).to(BF))
    # saturating E4M3 / E5M2
    v = torch.tensor([0.0, 1.0, -1.0, 447.0, 470.0, 1e6, -1e6, 2.0 ** -10])
    assert ref.fp8_saturate(v).view(torch.float8_e4m3fn).float().tolist()[3:7] == [448.0, 448.0, 448.0, -448.0]
    assert ref.fp8_saturate(v, True).view(torch.float8_e5m2).float().tolist()[5] == 57344.0
    # fp8_prep: an unrecorded site keeps its old estimate
    r = ref.fp8_prep_exact(torch.tensor([[2.0, 0.0], [2.0, 3.0]]), torch.tensor([0.5, 0.5]), 1.0, 1)
    assert r["state"].tolist() == [[2.0, 0.0], [3.0, 0.0]]
    assert r["inv_sx"][0].item() == pytest.approx(448.0 / 2.0) and r["inv_sx"][1].item() == pytest.approx(57344.0 / 3.0)


# ----------------------------------------------------------------------------------------------- the comparators reject defects
def _rms_bwd_case(M=1500, H=264):
    x, w, dy, rstd = _rms_inputs(M, H, 3)
    r = ref.rmsnorm_bwd_ref(dy, x, w, rstd, None, torch.ones(H))
    return x, w, dy, rstd, r


def test_a_correctly_rounded_result_passes():
    x, w, dy, rstd, r = _rms_bwd_case()
    assert ref.assert_rowwise_close("dx", r["dx"][0].to(BF), *r["dx"]) <= 1.0
    assert ref.assert_rowwise_close("dw", r["dw"][0].float(), *r["dw"]) <= 1.0


def test_one_perturbed_element_is_rejected():
    _, _, _, _, r = _rms_bwd_case()
    got = r["dx"][0].to(BF)
    got[17, 5] = (got[17, 5].float() * 1.02).to(BF)
    with pytest.raises(AssertionError, match=r"\(17, 5\)"):
        ref.assert_rowwise_close("dx", got, *r["dx"])


@pytest.mark.parametrize("fill", [float("nan"), 0.0])
def test_a_missing_last_vector_of_a_row_is_rejected(fill):
    _, _, _, _, r = _rms_bwd_case()
    got = r["dx"][0].to(BF)
    got[1499, -8:] = fill
    _fails(ref.assert_rowwise_close, "dx", got, *r["dx"])


def test_an_unwritten_element_is_rejected():
    x, w, _, rstd, _ = _rms_bwd_case()
    y = ref.rmsnorm_fwd_ref(x, w, 1e-5, rstd)["y"].clone()
    y[3, 100] = float("nan")
    _fails(ref.assert_bitwise_equal, "y", y, ref.rmsnorm_fwd_ref(x, w, 1e-5, rstd)["y"])
    _, _, _, _, r = _rms_bwd_case()
    got = r["dx"][0].to(BF)
    got[0, 0] = float("nan")
    _fails(ref.assert_rowwise_close, "dx", got, *r["dx"])


def test_an_unrounded_xhat_in_dw_is_rejected():
    """dw must sum dy·bf16(x̂); a kernel that sums dy·x̂ is off by ~2⁻⁹·√M per column, far above the fp32 accumulation bound."""
    x, w, dy, rstd, r = _rms_bwd_case()
    unrounded = 1.0 + (dy.float() * (x.float() * rstd[:, None])).sum(0)
    _fails(ref.assert_rowwise_close, "dw", unrounded, *r["dw"])


def test_a_missing_minus_one_at_a_tail_label_is_rejected():
    V = 1003
    x = (torch.randn(5, V, generator=_g(2)) * 2).to(BF)
    lab = torch.tensor([V - 2, 0, 4, V - 1, 17])  # V - 2 and V - 1 sit in the scalar tail (V % 8 = 3)
    r = ref.cross_entropy_ref(x, lab, V, 1.0, -100, torch.zeros(1), torch.zeros(1))
    got = r["grad"][0].to(BF)
    assert ref.assert_rowwise_close("grad", got, *r["grad"]) <= 1.0
    got[0, V - 2] = (got[0, V - 2].float() + 1.0).to(BF)
    with pytest.raises(AssertionError, match=rf"\(0, {V - 2}\)"):
        ref.assert_rowwise_close("grad", got, *r["grad"])


def test_ln_add_total_into_only_one_output_is_rejected():
    M, H = 64, 136
    g = _g(4)
    x = torch.randn(M, H, generator=g).to(BF)
    dy, dres = torch.randn(M, H, generator=g).to(BF), torch.randn(M, H, generator=g).to(BF)
    w = torch.ones(H).to(BF)
    mean, rstd = x.float().mean(-1), torch.rsqrt(x.float().var(-1, unbiased=False) + 1e-5)
    s1, s2 = torch.randn(H, generator=g), torch.randn(H, generator=g)
    r = ref.layernorm_bwd_ref(x, mean, rstd, [(dy, w, torch.zeros(H), None)], dres, (s1, s2))
    both = (s1.double() + dres.double().sum(0)).float()
    assert ref.assert_rowwise_close("dres_sum", both, *r["dres_sum0"]) <= 1.0
    _fails(ref.assert_rowwise_close, "dres_sum2", s2, *r["dres_sum1"])


def test_untouched_columns_must_keep_their_bits():
    T, hd, rot = 5, 64, 16
    cos, sin = (t.to(BF) for t in ref.rope_tables(rot, T))
    x = torch.randn(T, 3 * hd, generator=_g(6)).to(BF)
    mask, r, b = ref.rope_inplace_ref(x, T, 2, hd, rot, cos, sin, False, 0)
    got = r.to(BF)
    ref.assert_bitwise_equal("untouched", got[~mask], x[~mask])
    got[2, 2 * hd + 3] = 0.0  # a v column written
    _fails(ref.assert_bitwise_equal, "untouched", got[~mask], x[~mask])
    assert not math.isnan(ref.assert_rowwise_close("rotated", got[mask], r[mask], b[mask]))


# ----------------------------------------------------------------------------------------------- the audit's signature table
def _params(doc: str):
    """``[(name, default text or None)]`` of the first line of a pybind11 docstring ``f(a: T, b: T = d) -> R``."""
    head = doc.splitlines()[0]
    body = head[head.index("(") + 1:head.rindex(") ->")]
    parts, depth, cur = [], 0, ""
    for ch in body:
        depth += ch in "[(" and 1 or (ch in "])" and -1 or 0)
        if ch == "," and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += ch
    if cur.strip():
        parts.append(cur.strip())
    out = []
    for p in parts:
        name, _, rest = p.partition(":")
        out.append((name.strip(), rest.split(" = ", 1)[1].strip() if " = " in rest else None))
    return out


def test_the_audit_signature_table_matches_the_bindings():
    """tests/test_rowwise_modes_gpu.py binds the executors' positional arguments by a hand-written table of each entry point's
    parameters: its order, names and defaults must be the extension's (unnamed pybind parameters show as arg0, arg1, ...)."""
    import ast

    from test_rowwise_modes_gpu import _SIGS

    C = pytest.importorskip("relora_b200._C")
    for fn, (names, defaults) in _SIGS.items():
        got = _params(getattr(C, fn).__doc__)
        names = names.split()
        assert len(got) == len(names), f"{fn}: the extension takes {len(got)} parameters, the table lists {len(names)}"
        for i, ((gname, gdef), name) in enumerate(zip(got, names)):
            if gname != f"arg{i}":
                assert gname == name, f"{fn}: parameter {i} is {gname!r}, the table says {name!r}"
            assert (gdef is not None) == (name in defaults), f"{fn}: default of {name!r} differs"
            if gdef is not None:
                want = defaults[name]
                have = None if gdef == "None" else ast.literal_eval(gdef)
                assert (list(have) if isinstance(have, (list, tuple)) else have) == (
                    list(want) if isinstance(want, (list, tuple)) else want), f"{fn}: default of {name!r} is {gdef}"
