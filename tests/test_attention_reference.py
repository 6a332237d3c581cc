"""The fp64 reference of the wgmma attention kernels (ops/reference.py: attention_ref) and its comparator
assert_attention_close, on the CPU: the reference agrees with fp64 autograd of a plain masked softmax for multi-head,
grouped-query and interleaved layouts, its bounds are sane, and the tolerance rejects each structural defect a kernel could
have, at the shapes the GPU sweep (test_attention_modes_gpu.py) uses."""
import math

import pytest
import torch

from relora_b200.ops import reference as ref

BF, F64 = torch.bfloat16, torch.float64
LN2 = math.log(2.0)


def _qkv(B, T, nh, hd, nkv, seed, batch_scale=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * T, (nh + 2 * nkv) * hd, generator=g)
    if batch_scale:  # every batch at a different scale, so a row that leaks into the next batch is far off
        x = x * torch.arange(1, B + 1).repeat_interleave(T)[:, None]
    return x.to(BF)


def _dout(B, T, nh, hd, seed):
    return (torch.randn(B * T, nh * hd, generator=torch.Generator().manual_seed(seed)) * 0.5).to(BF)


def _plain(qkv, B, T, nh, hd, nkv, scale, interleaved, dout):
    """fp64 autograd of softmax(masked q·kᵀ·scale)·v over the packed buffer, indexing it independently of attention_unpack:
    returns (out [B*T, nh*hd], lse [B, nh, T], dqkv [B*T, W])."""
    x = qkv.to(F64).requires_grad_()
    if interleaved:
        cols = lambda h, part: slice((3 * h + part) * hd, (3 * h + part + 1) * hd)  # noqa: E731
        qc = [cols(h, 0) for h in range(nh)]
        kc = [cols(h, 1) for h in range(nh)]
        vc = [cols(h, 2) for h in range(nh)]
    else:
        qc = [slice(h * hd, (h + 1) * hd) for h in range(nh)]
        kc = [slice((nh + j) * hd, (nh + j + 1) * hd) for j in range(nkv)]
        vc = [slice((nh + nkv + j) * hd, (nh + nkv + j + 1) * hd) for j in range(nkv)]
    rows = x.view(B, T, -1)
    q = torch.stack([rows[:, :, c] for c in qc], 1)
    k = torch.stack([rows[:, :, c] for c in kc], 1).repeat_interleave(nh // len(kc), dim=1)
    v = torch.stack([rows[:, :, c] for c in vc], 1).repeat_interleave(nh // len(vc), dim=1)
    s = (q @ k.transpose(-1, -2)) * scale
    s = s.masked_fill(~torch.ones(T, T, dtype=torch.bool).tril(), -math.inf)
    o = torch.softmax(s, -1) @ v
    lse = torch.logsumexp(s, -1) / LN2
    o2 = o.transpose(1, 2).reshape(B * T, nh * hd)
    o2.backward(dout.to(F64))
    return o2.detach(), lse.detach(), x.grad


CASES = {  # (B, T, nh, hd, nkv, interleaved)
    "mha": (2, 129, 2, 40, 2, False),
    "gqa": (2, 77, 8, 16, 2, False),
    "mqa": (1, 65, 4, 24, 1, False),
    "interleaved": (3, 33, 3, 16, 3, True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_attention_ref_matches_fp64_autograd(case):
    B, T, nh, hd, nkv, il = CASES[case]
    scale = 0.3 if case == "mqa" else 1.0 / math.sqrt(hd)
    qkv, dout = _qkv(B, T, nh, hd, nkv, 1), _dout(B, T, nh, hd, 2)
    o, lse, dqkv = _plain(qkv, B, T, nh, hd, nkv, scale, il, dout)
    r = ref.attention_ref(qkv, B, T, nh, hd, scale, interleaved=il, nkv=nkv, out=o, dout=dout)
    kw = dict(nkv=nkv, interleaved=il)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)  # noqa: E731
    close(r["out"][0], ref.attention_heads(o, B, T, nh, hd))
    close(r["lse"][0], lse)
    for name, want in zip(("dq", "dk", "dv"), ref.attention_unpack(dqkv, B, T, nh, hd, **kw)):
        close(r[name][0], want)


def test_gqa_reference_is_the_repeated_kv_heads_summed_back():
    """attention_ref with nkv KV heads equals the multi-head reference on K / V repeated per query head, with dK / dV of the
    repeated heads summed back over each group."""
    B, T, nh, hd, nkv = 2, 70, 4, 16, 2
    group, scale = nh // nkv, 0.25
    qkv, dout = _qkv(B, T, nh, hd, nkv, 3), _dout(B, T, nh, hd, 4)
    q, k, v = ref.attention_unpack(qkv, B, T, nh, hd, nkv=nkv)
    rep = lambda t: t.repeat_interleave(group, dim=1).transpose(1, 2).reshape(B * T, nh * hd)  # noqa: E731
    mha = torch.cat([q.transpose(1, 2).reshape(B * T, nh * hd), rep(k), rep(v)], 1)
    fwd = ref.attention_ref(mha, B, T, nh, hd, scale)
    out = fwd["out"][0].transpose(1, 2).reshape(B * T, nh * hd).to(BF)
    a = ref.attention_ref(qkv, B, T, nh, hd, scale, nkv=nkv, out=out, dout=dout)
    b = ref.attention_ref(mha, B, T, nh, hd, scale, out=out, dout=dout)
    for name in ("out", "lse", "dq"):
        for x, y in zip(a[name], b[name]):
            torch.testing.assert_close(x, y, rtol=1e-12, atol=1e-12)
    for name in ("dk", "dv"):
        for x, y in zip(a[name], b[name]):
            torch.testing.assert_close(x, y.reshape(B, nkv, group, T, hd).sum(2), rtol=1e-12, atol=1e-12)


def test_interleaved_reference_is_a_permutation_of_the_default():
    B, T, nh, hd = 2, 45, 3, 24
    qkv, dout = _qkv(B, T, nh, hd, nh, 5), _dout(B, T, nh, hd, 6)
    il = qkv.view(B * T, 3, nh, hd).transpose(1, 2).reshape(B * T, 3 * nh * hd)  # [nh, (q|k|v), hd] per row
    out = ref.attention_ref(qkv, B, T, nh, hd, 0.2)["out"][0].transpose(1, 2).reshape(B * T, nh * hd).to(BF)
    a = ref.attention_ref(qkv, B, T, nh, hd, 0.2, out=out, dout=dout)
    b = ref.attention_ref(il, B, T, nh, hd, 0.2, interleaved=True, out=out, dout=dout)
    for name in a:
        for x, y in zip(a[name], b[name]):
            assert torch.equal(x, y), name
    for x, y in zip(ref.attention_unpack(qkv, B, T, nh, hd), ref.attention_unpack(il, B, T, nh, hd, interleaved=True)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("case", list(CASES))
def test_bounds_are_finite_and_cover_the_result(case):
    """Every bound is finite and >= 0; by the triangle inequality the out, dq, dk and dv bounds are >= |ref|; the flush floor
    stays at the scale of the smallest normal fp32."""
    B, T, nh, hd, nkv, il = CASES[case]
    qkv, dout = _qkv(B, T, nh, hd, nkv, 7), _dout(B, T, nh, hd, 8)
    out = ref.attention_ref(qkv, B, T, nh, hd, 0.5, interleaved=il, nkv=nkv)["out"][0]
    out = out.transpose(1, 2).reshape(B * T, nh * hd).to(BF)
    r = ref.attention_ref(qkv, B, T, nh, hd, 0.5, interleaved=il, nkv=nkv, out=out, dout=dout)
    for name, (val, bound, score, floor) in r.items():
        for t in (bound, score, floor):
            assert bool(torch.isfinite(t).all() and (t >= 0).all()), name
        assert float(floor.max()) < 1e-30, name
        if name != "lse":
            assert bool((bound >= val.abs() * (1 - 1e-12)).all()), name


def test_results_below_the_fp32_normal_range_may_flush_to_zero():
    """Scores in the hundreds of nats leave dK / dV elements far below 2⁻¹²⁶, which the kernels' FTZ arithmetic returns as 0."""
    B, T, nh, hd = 1, 129, 1, 64
    g = torch.Generator().manual_seed(9)
    qkv = (torch.randn(B * T, 3 * nh * hd, generator=g) * torch.tensor([10.0] * 2 * hd + [1.0] * hd)).to(BF)
    out = ref.attention_ref(qkv, B, T, nh, hd, 0.125)["out"][0].transpose(1, 2).reshape(B * T, nh * hd).to(BF)
    r = ref.attention_ref(qkv, B, T, nh, hd, 0.125, out=out, dout=_dout(B, T, nh, hd, 10))
    for name in ("dk", "dv"):
        val = r[name][0]
        tiny = (val != 0) & (val.abs() < 2.0 ** -126)
        assert bool(tiny.any()), name
        ref.assert_attention_close(name, torch.where(tiny, 0.0, val).to(BF), *r[name])


# ----------------------------------------------------------------------------------------------- teeth
def _expected(r, name):
    return r[name][0].to(torch.float32 if name == "lse" else BF)


def _fails(name, got, r):
    with pytest.raises(AssertionError, match=f"attention {name} out of tolerance"):
        ref.assert_attention_close(name, got, *r[name])


def _attn(q, k, v, scale, mask):
    """fp64 (out, lse) of one head-batched q [.., T, hd] against k, v [.., S, hd] under a [T, S] mask."""
    s = (scale * (q @ k.transpose(-1, -2))).masked_fill(~mask, -math.inf)
    return torch.softmax(s, -1) @ v, torch.logsumexp(s, -1) / LN2


SWEEP = [(2, 129, 2, 64, 2), (3, 1000, 1, 64, 1), (2, 129, 8, 64, 2), (2, 33, 4, 128, 1)]  # (B, T, nh, hd, nkv) of the GPU sweep


def _fwd_case(B, T, nh, hd, nkv, seed):
    qkv = _qkv(B, T, nh, hd, nkv, seed, batch_scale=True)
    q, k, v = (t.to(F64) for t in ref.attention_unpack(qkv, B, T, nh, hd, nkv=nkv))
    kvh = torch.arange(nh) // (nh // nkv)
    return qkv, q, k[:, kvh], v[:, kvh], ref.attention_ref(qkv, B, T, nh, hd, 1.0 / math.sqrt(hd), nkv=nkv)


@pytest.mark.parametrize("shape", SWEEP)
def test_comparator_accepts_the_rounded_reference(shape):
    """The control of the defect tests below: the reference itself, rounded to the kernels' output types, passes."""
    B, T, nh, hd, nkv = shape
    qkv, q, kr, vr, r = _fwd_case(B, T, nh, hd, nkv, 11)
    for name in ("out", "lse"):
        assert ref.assert_attention_close(name, _expected(r, name), *r[name]) <= 1.0


@pytest.mark.parametrize("defect", ["mask_shift", "diagonal_dropped"])
@pytest.mark.parametrize("shape", SWEEP)
def test_comparator_rejects_a_wrong_causal_mask(shape, defect):
    B, T, nh, hd, nkv = shape
    qkv, q, kr, vr, r = _fwd_case(B, T, nh, hd, nkv, 12)
    ones = torch.ones(T, T, dtype=torch.bool)
    if defect == "mask_shift":  # query i also sees key i + 1
        mask = ones.tril(1)
    else:  # query i no longer sees key i (row 0 keeps its only key, so the row stays finite)
        mask = ones.tril(-1)
        mask[0, 0] = True
    o, lse = _attn(q, kr, vr, 1.0 / math.sqrt(hd), mask)
    _fails("out", o.to(BF), r)
    _fails("lse", lse.float(), r)


@pytest.mark.parametrize("B,T", [(2, 129), (3, 1000), (2, 65), (3, 17)])
def test_comparator_rejects_the_next_batch_leaking_into_the_tail_rows(B, T):
    """The rows of the last 64-row query tile of batch b < B - 1 also see key 0 of batch b + 1 (the tile runs into those rows)."""
    nh = nkv = 1
    hd = 64
    qkv, q, kr, vr, r = _fwd_case(B, T, nh, hd, nkv, 13)
    mask = torch.ones(T, T + 1, dtype=torch.bool)
    mask[:, :T] = torch.ones(T, T, dtype=torch.bool).tril()
    mask[: (T - 1) // 64 * 64, T] = False
    o, lse = _attn(q, kr, vr, 1.0 / math.sqrt(hd), torch.ones(T, T, dtype=torch.bool).tril())
    o, lse = o.clone(), lse.clone()
    for b in range(B - 1):
        kx = torch.cat([kr[b], kr[b + 1, :, :1]], 1)
        vx = torch.cat([vr[b], vr[b + 1, :, :1]], 1)
        o[b], lse[b] = _attn(q[b], kx, vx, 1.0 / math.sqrt(hd), mask)
    _fails("out", o.to(BF), r)


@pytest.mark.parametrize("shape", SWEEP)
def test_comparator_rejects_lse_in_the_natural_log_domain(shape):
    B, T, nh, hd, nkv = shape
    qkv, q, kr, vr, r = _fwd_case(B, T, nh, hd, nkv, 14)
    _fails("lse", (r["lse"][0] * LN2).float(), r)


def _rising(B, T, nh, hd, nkv, seed):
    """Scores that rise with the key index: every 64-key block raises each row's running maximum."""
    g = torch.Generator().manual_seed(seed)
    W = (nh + 2 * nkv) * hd
    x = torch.randn(B * T, W, generator=g) * 0.3
    x4 = x.view(B, T, nh + 2 * nkv, hd)
    x4[:, :, :nh, 0] = 1.0
    x4[:, :, nh:nh + nkv, 0] = torch.arange(T, dtype=torch.float32).view(1, T, 1) * (4.0 / 64)
    return x.to(BF)


@pytest.mark.parametrize("B,T,nh,hd,nkv", [(2, 1000, 2, 64, 2), (2, 129, 4, 128, 1)])
def test_comparator_rejects_a_missing_corr_rescale(B, T, nh, hd, nkv):
    """The online softmax without o *= corr: the accumulated P·V of earlier key blocks keeps the old running maximum."""
    qkv = _rising(B, T, nh, hd, nkv, 15)
    scale = 1.0 / math.sqrt(hd)
    r = ref.attention_ref(qkv, B, T, nh, hd, scale, nkv=nkv)
    q, k, v = (t.to(F64) for t in ref.attention_unpack(qkv, B, T, nh, hd, nkv=nkv))
    kvh = torch.arange(nh) // (nh // nkv)
    kr, vr = k[:, kvh], v[:, kvh]
    s = (scale * (q @ kr.transpose(-1, -2))).masked_fill(~torch.ones(T, T, dtype=torch.bool).tril(), -math.inf)
    o = torch.zeros_like(q)
    m = torch.full(q.shape[:-1] + (1,), -math.inf, dtype=F64)
    l = torch.zeros_like(m)
    for k0 in range(0, T, 64):
        sb = s[..., k0:k0 + 64]
        mx = torch.maximum(m, sb.amax(-1, keepdim=True))
        live = torch.isfinite(mx)
        corr = torch.where(live, torch.exp(m - mx), 1.0)
        p = torch.where(live, torch.exp(sb - mx), 0.0)
        o = o + p @ vr[..., k0:k0 + 64, :]  # the defect: o is not multiplied by corr
        l = l * corr + p.sum(-1, keepdim=True)
        m = torch.where(live, mx, m)
    _fails("out", (o / l).to(BF), r)


@pytest.mark.parametrize("B,T,nh,hd,nkv", [(2, 129, 8, 64, 2), (2, 1000, 4, 128, 1), (2, 129, 2, 64, 1)])
def test_comparator_rejects_a_query_head_missing_from_one_key_block_of_dk_dv(B, T, nh, hd, nkv):
    """KV head 0, keys 64..127: dK / dV lack the last query head of the group."""
    group, scale = nh // nkv, 1.0 / math.sqrt(hd)
    qkv, dout = _qkv(B, T, nh, hd, nkv, 16), _dout(B, T, nh, hd, 17)
    out = ref.attention_ref(qkv, B, T, nh, hd, scale, nkv=nkv)["out"][0].transpose(1, 2).reshape(B * T, nh * hd).to(BF)
    r = ref.attention_ref(qkv, B, T, nh, hd, scale, nkv=nkv, out=out, dout=dout)
    # the same backward with that head's dout zeroed, for KV head 0's keys 64..127 only
    d0 = dout.clone()
    d0.view(B, T, nh, hd)[:, :, group - 1] = 0
    r0 = ref.attention_ref(qkv, B, T, nh, hd, scale, nkv=nkv, out=out, dout=d0)
    for name in ("dk", "dv"):
        got = r[name][0].clone()
        got[:, 0, 64:128] = r0[name][0][:, 0, 64:128]
        _fails(name, got.to(BF), r)
