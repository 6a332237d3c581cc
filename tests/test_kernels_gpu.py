"""Numerics of the sm_90a kernels against plain PyTorch fp32 references (run on an H100: -m gpu)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


@pytest.fixture(scope="module")
def F():
    from relora_b200.ops import fused

    return fused


def _rand(*shape, scale=1.0, device="cuda"):
    return (torch.randn(*shape, device=device, dtype=torch.float32) * scale).to(BF)


def _relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp(min=1e-12))


# ----------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K,block_n", [
    (128, 128, 64, 128), (256, 256, 128, 128), (384, 768, 768, 128), (1000, 520, 200, 128),
    (512, 1024, 512, 256), (640, 2304, 768, 256), (130, 264, 72, 0), (2048, 2560, 768, 0),
])
def test_gemm_kmajor(F, M, N, K, block_n):
    torch.manual_seed(0)
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    out = F.gemm(a, b, block_n=block_n)
    ref = a.float() @ b.float().t()
    assert out.shape == (M, N)
    assert _relerr(out, ref) < 6e-3


def test_gemm_residual_alpha_accumulate_f32(F):
    torch.manual_seed(1)
    M, N, K = 384, 512, 256
    a, b, r = _rand(M, K), _rand(N, K, scale=0.05), _rand(M, N)
    out = F.gemm(a, b, residual=r, alpha=0.5)
    ref = 0.5 * (a.float() @ b.float().t()) + r.float()
    assert _relerr(out, ref) < 6e-3
    acc = torch.randn(M, N, device="cuda", dtype=torch.float32)
    want = acc + a.float() @ b.float().t()
    F.gemm(a, b, acc, accumulate=True)
    assert _relerr(acc, want) < 1e-3
    accb = _rand(M, N)
    wantb = accb.float() + 2.0 * (a.float() @ b.float().t())
    F.gemm(a, b, accb, accumulate=True, alpha=2.0)
    assert _relerr(accb, wantb) < 6e-3


@pytest.mark.parametrize("G,Ng,K,r,block_n", [(1, 768, 768, 128, 128), (3, 768, 768, 128, 128), (2, 2560, 768, 128, 256),
                                               (3, 256, 320, 64, 128), (1, 768, 2560, 128, 256)])
def test_gemm_fused_lora_groups(F, G, Ng, K, r, block_n):
    """y_g = x W_gᵀ + u_g B_gᵀ in one launch: the LoRA up-projection as extra K iterations."""
    torch.manual_seed(2)
    M, N = 640, G * Ng
    x, W = _rand(M, K), _rand(N, K, scale=0.03)
    u, B = _rand(M, G * r), _rand(N, r, scale=0.05)
    out = F.gemm(x, W, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, block_n=block_n)
    ref = x.float() @ W.float().t()
    for g in range(G):
        ref[:, g * Ng:(g + 1) * Ng] += u[:, g * r:(g + 1) * r].float() @ B[g * Ng:(g + 1) * Ng].float().t()
    assert _relerr(out, ref) < 6e-3


@pytest.mark.parametrize("block_n", [128, 256, 0])
def test_gemm_ragged_groups_and_tma_residual(F, block_n):
    """Groups whose width is a multiple of 64 but not of the tile (llama_1b: 5504): the last tile of a group is
    ragged.  Also exercises the residual fetched by TMA into the output slab."""
    torch.manual_seed(3)
    M, K, G, Ng, r = 300, 192, 2, 320, 128
    x, W = _rand(M, K), _rand(G * Ng, K, scale=0.05)
    u, B = _rand(M, G * r), _rand(G * Ng, r, scale=0.05)
    res = _rand(M, G * Ng)
    out = torch.full((M, G * Ng), 7.0, device="cuda", dtype=BF)
    F.gemm(x, W, out, M=M, N=G * Ng, K1=K, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, residual=res, block_n=block_n)
    want = x.float() @ W.float().t() + res.float()
    for g in range(G):
        want[:, g * Ng:(g + 1) * Ng] += u[:, g * r:(g + 1) * r].float() @ B[g * Ng:(g + 1) * Ng].float().t()
    assert _relerr(out, want) < 5e-3
    # plain residual GEMM with ragged M / N edges
    M, N, K = 1000, 520, 200
    a, b, res = _rand(M, K), _rand(N, K, scale=0.05), _rand(M, N)
    out = torch.empty(M, N, device="cuda", dtype=BF)
    F.gemm(a, b, out, residual=res, block_n=block_n)
    assert _relerr(out, a.float() @ b.float().t() + res.float()) < 5e-3


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [
    (512, 512, 256, False, False), (1000, 520, 200, False, False), (768, 1024, 384, False, True), (640, 768, 320, True, True),
    (384, 256, 192, True, False), (12288, 2304, 768, False, False),
])
def test_gemm_cta_pair(F, M, N, K, a_mn, b_mn):
    """The CTA-pair request of the Blackwell build is accepted on sm_90 (no cta_group::2 MMA there) and computes the same product."""
    torch.manual_seed(M + N)
    a = _rand(K, M) if a_mn else _rand(M, K)
    b = _rand(K, N, scale=0.05) if b_mn else _rand(N, K, scale=0.05)
    out = torch.empty(M, (N + 7) // 8 * 8, device="cuda", dtype=BF)[:, :N]
    F.gemm(a, b, out, M=M, N=N, K1=K, a1_mn=a_mn, b1_mn=b_mn, block_n=256, pair=1)
    af = a.float().t() if a_mn else a.float()
    bf = b.float() if b_mn else b.float().t()
    assert _relerr(out, af @ bf) < 5e-3


def test_gemm_cta_pair_fused_lora_residual_splitk(F):
    torch.manual_seed(11)
    M, K, G, Ng, r = 700, 256, 2, 512, 128
    x, W = _rand(M, K), _rand(G * Ng, K, scale=0.05)
    u, B = _rand(M, G * r), _rand(G * Ng, r, scale=0.05)
    res = _rand(M, G * Ng)
    out = torch.empty(M, G * Ng, device="cuda", dtype=BF)
    F.gemm(x, W, out, M=M, N=G * Ng, K1=K, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, residual=res, block_n=256, pair=1)
    want = x.float() @ W.float().t() + res.float()
    for g in range(G):
        want[:, g * Ng:(g + 1) * Ng] += u[:, g * r:(g + 1) * r].float() @ B[g * Ng:(g + 1) * Ng].float().t()
    assert _relerr(out, want) < 5e-3
    # weight-gradient shape: fp32 accumulate with split-K over the tokens
    dy, xx = _rand(4096, 512), _rand(4096, 256)
    dw = torch.ones(512, 256, device="cuda", dtype=torch.float32)
    F.gemm(dy, xx, dw, M=512, N=256, K1=4096, a1_mn=True, b1_mn=True, accumulate=True, split_k=8, block_n=256, pair=1)
    assert _relerr(dw, 1.0 + dy.float().t() @ xx.float()) < 5e-3


def test_gemm_grouped_a1_window(F):
    """u_g = xd_g A_gᵀ for G groups at once (per-group K window of A1)."""
    torch.manual_seed(3)
    M, K, r, G = 512, 768, 128, 3
    xd, A = _rand(M, G * K), _rand(G * r, K, scale=0.05)
    out = F.gemm(xd, A, M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K, alpha=0.25)
    ref = torch.cat([0.25 * xd[:, g * K:(g + 1) * K].float() @ A[g * r:(g + 1) * r].float().t() for g in range(G)], 1)
    assert _relerr(out, ref) < 6e-3


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K,block_n", [(256, 256, 128, 128), (768, 128, 1024, 128), (384, 512, 320, 256), (200, 136, 96, 128)])
def test_gemm_mn_major(F, a_mn, b_mn, M, N, K, block_n):
    torch.manual_seed(4)
    a, b = _rand(M, K), _rand(N, K, scale=0.05)
    a_in = a.t().contiguous() if a_mn else a
    b_in = b.t().contiguous() if b_mn else b
    out = F.gemm(a_in, b_in, M=M, N=N, K1=K, a1_mn=a_mn, b1_mn=b_mn, block_n=block_n)
    ref = a.float() @ b.float().t()
    assert _relerr(out, ref) < 6e-3


@pytest.mark.parametrize("split", [0, 2, 7])
def test_gemm_split_k_weight_grad(F, split):
    """dA[r, K] = duᵀ · xd: reduction over tokens, both operands MN-major, fp32 atomics."""
    torch.manual_seed(5)
    Mtok, r, K = 4096, 128, 768
    du, xd = _rand(Mtok, r, scale=0.1), _rand(Mtok, K)
    out = torch.zeros(r, K, device="cuda", dtype=torch.float32)
    F.gemm(du, xd, out, M=r, N=K, K1=Mtok, a1_mn=True, b1_mn=True, accumulate=True, split_k=split)
    ref = du.float().t() @ xd.float()
    assert _relerr(out, ref) < 2e-3


def test_gemm_many_tiles_persistent(F):
    torch.manual_seed(6)
    M, N, K = 4096, 2304, 768  # 576 tiles of 128x128 > 132 SMs: exercises the ring phases
    a, b = _rand(M, K), _rand(N, K, scale=0.03)
    out = F.gemm(a, b, block_n=128)
    assert _relerr(out, a.float() @ b.float().t()) < 6e-3
    out2 = F.gemm(a, b, block_n=256)
    assert _relerr(out2, a.float() @ b.float().t()) < 6e-3


@pytest.mark.parametrize("G,Ng,K,M,p", [(1, 256, 256, 300, 0.1), (2, 384, 256, 512, 0.1), (3, 256, 384, 1000, 0.1), (3, 128, 128, 128, 0.0),
                                        (1, 256, 640, 20000, 0.25), (2, 5504, 2048, 256, 0.1)])
def test_lora_dx_fused_dropout_epilogue(C, G, Ng, K, M, p):
    """dx = dy·W + Σ_g keep_g ⊙ (du_g·A_g)/(1-p): masked LoRA terms folded into the register accumulator."""
    from relora_b200.ops import reference as ref

    r = 128
    torch.manual_seed(G * 7 + M)
    dy, W = _rand(M, G * Ng), _rand(G * Ng, K, scale=0.05)
    du, A = _rand(M, G * r), _rand(G * r, K, scale=0.05)
    seed = torch.tensor([1234567], dtype=torch.int32, device="cuda")
    keys = [11, 22, 33][:G]
    out = torch.empty(M, K, dtype=BF, device="cuda")
    C.lora_dx(dy, W, du, A, out, seed if p > 0 else None, keys, p)
    want = dy.float() @ W.float()
    for g in range(G):
        part = du[:, g * r:(g + 1) * r].float() @ A[g * r:(g + 1) * r].float()
        if p > 0:
            keep = ref.dropout_keep_mask(ref.mix_seed(1234567, keys[g]), M, K, p, device="cuda")
            part = part * keep / (1.0 - p)
        want = want + part
    assert _relerr(out, want) < 6e-3
    # two-kernel form: the frozen-path product comes from the plain GEMM, this kernel only adds the masked terms
    base = (dy.float() @ W.float()).to(BF)
    out2 = torch.empty_like(out)
    C.lora_dx(None, None, du, A, out2, seed if p > 0 else None, keys, p, base)
    assert _relerr(out2, want) < 8e-3
    # the mask really is applied per group: without it the result differs by O(p)
    if p > 0:
        nomask = dy.float() @ W.float() + du.float() @ A.float() / (1.0 - p)
        assert _relerr(out, nomask) > 1e-2


# ----------------------------------------------------------------------------------------- elementwise
@pytest.mark.parametrize("M,H", [(64, 768), (300, 2048), (17, 4096), (5, 128)])
def test_rmsnorm_fwd_bwd(C, M, H):
    from relora_b200.ops import reference as ref

    torch.manual_seed(0)
    x, w = _rand(M, H), (1 + 0.1 * torch.randn(H, device="cuda")).to(BF)
    y = torch.empty_like(x)
    rstd = torch.empty(M, device="cuda", dtype=torch.float32)
    C.rmsnorm_fwd(x, w, y, rstd, 1e-6, None, None, [], 0.0)
    want = ref.rmsnorm(x, w, 1e-6)
    assert _relerr(y, want) < 4e-3
    # backward vs autograd of the fp32 definition
    xf, wf = x.float().requires_grad_(), w.float().requires_grad_()
    dy = _rand(M, H)
    ref.rmsnorm_fp32(xf, wf, 1e-6).backward(dy.float())
    dx = torch.empty_like(x)
    dw = torch.zeros(H, device="cuda", dtype=torch.float32)
    from relora_b200.ops import fused

    ws, tk = fused.norm_workspace(x.device, H)
    C.rmsnorm_bwd(dy, x, w, rstd, None, dx, dw, ws, tk)
    dx2, dw2 = torch.empty_like(x), torch.zeros(H, device="cuda", dtype=torch.float32)
    C.rmsnorm_bwd(dy, x, w, rstd, None, dx2, dw2, None, None)  # block-per-row fallback
    assert _relerr(dx2, dx) < 1e-3 and _relerr(dw2, dw) < 1e-3
    assert _relerr(dx, xf.grad) < 1e-2
    assert _relerr(dw, wf.grad) < 1e-2


def test_dropout_mask_matches_reference_hash(C):
    from relora_b200.ops import reference as ref

    M, H, p = 96, 256, 0.1
    x = torch.ones(M, H, device="cuda", dtype=BF)
    seed = torch.tensor([12345], dtype=torch.int32, device="cuda")
    keys = [3, 11]
    xd = torch.empty(M, 2 * H, device="cuda", dtype=BF)
    C.dropout_expand(x, xd, seed, keys, p)
    for g, k in enumerate(keys):
        keep = ref.dropout_keep_mask(ref.mix_seed(12345, k), M, H, p, device="cuda")
        got = xd.view(M, 2, H)[:, g] != 0
        assert torch.equal(got, keep)
        assert abs(float(keep.float().mean()) - 0.9) < 0.02
    kept_vals = xd[xd != 0].float()
    assert torch.allclose(kept_vals, torch.full_like(kept_vals, 1 / 0.9), atol=1e-2)
    # combine = base + mask * part / (1-p)
    base, part = _rand(M, H), _rand(M, H)
    out = torch.empty_like(base)
    C.dropout_combine(base, part.reshape(1, M, H), out, seed, [keys[0]], p)
    keep = ref.dropout_keep_mask(ref.mix_seed(12345, keys[0]), M, H, p, device="cuda")
    want = base.float() + keep * part.float() / 0.9
    assert _relerr(out, want) < 5e-3


@pytest.mark.parametrize("hd,rot", [(48, 48), (64, 64), (64, 16), (128, 128)])
def test_rope_fwd_bwd(C, hd, rot):
    from relora_b200.ops import reference as ref

    torch.manual_seed(0)
    B, T, nh = 2, 40, 6
    buf = _rand(B * T, 3 * nh * hd)
    cos, sin = ref.rope_tables(rot, 64, device="cuda", dtype=BF)
    orig = buf.clone()
    C.rope_inplace(buf, T, 2 * nh, hd, rot, cos, sin, False, 0)
    x = orig.view(B, T, 3 * nh, hd).float()
    want = x.clone()
    want[:, :, : 2 * nh, :rot] = ref.rope_apply(x[:, :, : 2 * nh, :rot].transpose(1, 2), cos[:T].float(), sin[:T].float()).transpose(1, 2)
    assert _relerr(buf.view(B, T, 3 * nh, hd), want) < 5e-3
    assert torch.equal(buf.view(B, T, 3 * nh, hd)[:, :, 2 * nh:], orig.view(B, T, 3 * nh, hd)[:, :, 2 * nh:])
    # backward is the inverse rotation
    C.rope_inplace(buf, T, 2 * nh, hd, rot, cos, sin, True, 0)
    assert _relerr(buf, orig) < 1.5e-2


@pytest.mark.parametrize("hd,rot", [(48, 48), (64, 64), (64, 16)])
def test_rope_pack_bwd(C, hd, rot):
    from relora_b200.ops import reference as ref

    torch.manual_seed(1)
    B, T, nh = 2, 24, 4
    cos, sin = ref.rope_tables(rot, 32, device="cuda", dtype=BF)
    # gradients as attention backward returns them: [B, nh, T, hd] views of [B, T, nh, hd] memory
    dq, dk, dv = (_rand(B, T, nh, hd).transpose(1, 2) for _ in range(3))
    out = torch.empty(B * T, 3 * nh * hd, device="cuda", dtype=BF)
    C.rope_pack_bwd(dq, dk, dv, out, rot, cos, sin, 0)
    want = torch.empty_like(out)
    w5 = want.view(B, T, 3, nh, hd)
    w5[:, :, 0].copy_(dq.transpose(1, 2)); w5[:, :, 1].copy_(dk.transpose(1, 2)); w5[:, :, 2].copy_(dv.transpose(1, 2))
    C.rope_inplace(want, T, 2 * nh, hd, rot, cos, sin, True, 0)
    assert _relerr(out, want) < 1e-6
    # contiguous [B, nh, T, hd] inputs work too
    out2 = torch.empty_like(out)
    C.rope_pack_bwd(dq.contiguous(), dk.contiguous(), dv.contiguous(), out2, rot, cos, sin, 0)
    assert torch.equal(out, out2)


def test_swiglu(C):
    torch.manual_seed(0)
    M, Fd = 200, 2560
    gu = _rand(M, 2 * Fd)
    h = torch.empty(M, Fd, device="cuda", dtype=BF)
    C.swiglu_fwd(gu, h)
    g, u = gu[:, :Fd].float().requires_grad_(), gu[:, Fd:].float().requires_grad_()
    want = torch.nn.functional.silu(g) * u
    assert _relerr(h, want) < 5e-3
    dh = _rand(M, Fd)
    want.backward(dh.float())
    dgu = torch.empty_like(gu)
    C.swiglu_bwd(dh, gu, dgu)
    assert _relerr(dgu[:, :Fd], g.grad) < 6e-3 and _relerr(dgu[:, Fd:], u.grad) < 6e-3
    # fused dropout-expanded copy == dropout_expand(h) bit for bit
    seed = torch.tensor([777], dtype=torch.int32, device="cuda")
    h2, hd, hd_ref = torch.empty_like(h), torch.empty_like(h), torch.empty_like(h)
    C.swiglu_fwd(gu, h2, hd, seed, 5, 0.1)
    C.dropout_expand(h, hd_ref, seed, [5], 0.1)
    assert torch.equal(h2, h) and torch.equal(hd, hd_ref)


def test_embedding(C):
    torch.manual_seed(0)
    V, H, M = 1000, 256, 700
    table = _rand(V, H)
    ids = torch.randint(0, V, (M,), device="cuda")
    ids[:5] = V - 1
    out = torch.empty(M, H, device="cuda", dtype=BF)
    C.embedding_fwd(ids, table, out)
    assert torch.equal(out, table[ids])
    dout = _rand(M, H)
    dt = torch.zeros(V, H, device="cuda", dtype=torch.float32)
    C.embedding_bwd(ids, dout, dt, V - 1)
    want = torch.zeros(V, H, device="cuda").index_add_(0, ids, dout.float())
    want[V - 1] = 0
    assert _relerr(dt, want) < 1e-5
    # deterministic variant (stable sort, one writer per row): same values, bit-identical across repetitions and when
    # accumulating on top of an existing gradient
    sid, perm = torch.sort(ids, stable=True)
    runs = []
    for _ in range(3):
        d2 = torch.full((V, H), 0.25, device="cuda", dtype=torch.float32)
        C.embedding_bwd_sorted(sid, perm, dout, d2, V - 1)
        runs.append(d2)
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2])
    assert _relerr(runs[0] - 0.25, want) < 1e-5
    assert float(runs[0][V - 1].sub(0.25).abs().max()) == 0.0


@pytest.mark.parametrize("V", [32100, 1000, 50257])
def test_cross_entropy_in_place(C, V):
    torch.manual_seed(0)
    M = 64
    ld = (V + 7) // 8 * 8
    buf = torch.zeros(M, ld, device="cuda", dtype=BF)
    logits = buf[:, :V]
    logits.copy_(_rand(M, V, scale=2.0))
    labels = torch.randint(0, V, (M,), device="cuda")
    labels[3] = -100
    lf = logits.float().clone().requires_grad_()
    want = torch.nn.functional.cross_entropy(lf, labels, reduction="sum", ignore_index=-100)
    want.backward()
    loss, cnt = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    C.cross_entropy_fwd_bwd(logits, labels, V, 1.0, -100, loss, cnt)
    assert abs(float(loss) - float(want)) / float(want) < 2e-3
    assert float(cnt) == M - 1
    assert _relerr(logits, lf.grad) < 1e-2
    assert float(logits[3].abs().sum()) == 0


def test_lm_head_ce_function(F):
    from relora_b200.ops import reference as ref

    torch.manual_seed(0)
    B, T, H, V = 3, 65, 256, 32100
    h = _rand(B, T, H).requires_grad_()
    w = _rand(V, H, scale=0.05).requires_grad_()
    labels = torch.randint(0, V, (B, T), device="cuda")
    loss = F.lm_head_cross_entropy(h, w, labels, chunk=100)
    loss.backward()
    hf, wf = h.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    want = ref.lm_head_cross_entropy(hf, wf, labels)
    want.backward()
    assert abs(float(loss) - float(want)) < 5e-3
    assert _relerr(h.grad, hf.grad) < 2e-2
    assert _relerr(w.grad, wf.grad) < 2e-2


# ----------------------------------------------------------------------------------------- optimizer
@pytest.mark.parametrize("gdt,sdt", [(BF, BF), (torch.float32, BF), (torch.float32, torch.float32)])
def test_adamw_flat(C, gdt, sdt):
    from relora_b200.ops import reference as ref

    torch.manual_seed(0)
    n = 8 * 1000
    p = _rand(n)
    g = torch.randn(n, device="cuda").to(gdt)
    m = (0.1 * torch.randn(n, device="cuda")).to(sdt)
    v = (0.01 * torch.rand(n, device="cuda")).to(sdt)
    p2, m2, v2 = p.clone(), m.clone(), v.clone()
    gs = torch.tensor([0.5], device="cuda")
    # the bias corrections come from the device-resident step count (7) when one is passed; the host value (99) is then ignored
    step_dev = torch.tensor([7.0], device="cuda")
    C.adamw_flat(p, g, m, v, 1e-2, 0.9, 0.95, 1e-8, 0.01, 99, gs, 1.0, None, step_dev)
    ref.adamw_step(p2, g, m2, v2, step=7, lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.01, grad_scale=0.5)
    assert _relerr(p, p2) < 1e-3 and _relerr(m, m2) < 4e-3 and _relerr(v, v2) < 4e-3
    # device-side skip leaves everything untouched
    before, mb, vb = p.clone(), m.clone(), v.clone()
    C.adamw_flat(p, g, m, v, 1e-2, 0.9, 0.95, 1e-8, 0.01, 8, None, 1.0, torch.ones(1, device="cuda"), None)
    assert torch.equal(before, p)
    # ... and so does a non-finite gradient scale (= non-finite gradient norm upstream of the kernel)
    for bad in (float("nan"), float("inf")):
        C.adamw_flat(p, g, m, v, 1e-2, 0.9, 0.95, 1e-8, 0.01, 8, torch.tensor([bad], device="cuda"), 1.0, None, None)
        assert torch.equal(before, p) and torch.equal(mb, m) and torch.equal(vb, v)


def test_sumsq_and_pruning(C):
    from relora_b200.ops import reference as ref
    from relora_b200.relora.optim_reset import magnitude_pruning_

    torch.manual_seed(0)
    x = _rand(100_003)
    out = torch.zeros(1, device="cuda")
    C.sumsq(x, out)
    assert abs(float(out) - float(x.float().pow(2).sum())) / float(out) < 1e-4
    # random pruning == reference hash
    y = torch.ones(50_000, device="cuda", dtype=BF)
    C.random_prune(y, 0.999, 777, 5)
    keep = ref.random_prune_keep_mask(777, 50_000, 0.999, device="cuda", offset=5)
    assert torch.equal(y != 0, keep)
    # magnitude pruning == torch.quantile semantics, bf16 and fp32
    ws = torch.empty(C.quantile_workspace_bytes(), dtype=torch.uint8, device="cuda")
    thr = torch.zeros(1, device="cuda")
    for dt in (BF, torch.float32):
        z = (torch.randn(300_000, device="cuda") * 1e-3).to(dt)
        want = z.clone()
        magnitude_pruning_(want, 0.9)
        C.magnitude_prune(z, 0.9, ws, thr)
        assert torch.equal(z, want), dt


def test_transpose_and_fill(C):
    from relora_b200.ops import reference as ref

    a = _rand(100, 72)
    out = torch.empty(72, 100, device="cuda", dtype=BF)
    C.transpose(a, out)
    assert torch.equal(out, a.t())
    w = torch.empty(128, 768, device="cuda", dtype=BF)
    C.fill_uniform_hash(w, 4242, 1 / math.sqrt(768))
    want = ref.kaiming_uniform_from_hash(4242, 128, 768, 1 / math.sqrt(768), device="cuda").to(BF)
    assert torch.equal(w, want)
    assert float(w.float().abs().max()) <= 1 / math.sqrt(768) + 1e-4


# ----------------------------------------------------------------------------------------- module path
def test_relora_linear_fused_matches_reference():
    from relora_b200.ops import dispatch
    from relora_b200.ops import fused
    from relora_b200.ops import reference as ref
    from relora_b200.relora import ReLoRaLinear

    torch.manual_seed(0)
    lin = ReLoRaLinear(768, 2304, r=128, lora_alpha=32, lora_dropout=0.1, bias=False).cuda().to(BF)
    lin.weight.data.normal_(std=0.02)
    lin.lora_B.weight.data.normal_(std=0.02)
    lin.module_index = 4
    x = _rand(4, 96, 768).requires_grad_()
    fused.seed_state.set(x.device, 99)
    lin.train()
    y = lin(x)
    dy = _rand(4, 96, 2304, scale=0.1)
    y.backward(dy)
    seed = ref.mix_seed(99, 5)
    xf = x.detach().float().requires_grad_()
    Af, Bf = lin.lora_A.weight.detach().float().requires_grad_(), lin.lora_B.weight.detach().float().requires_grad_()
    want = ref.lora_linear(xf, lin.weight.float(), None, Af, Bf, lin.scaling, p=0.1, seed=seed)
    want.backward(dy.float())
    assert _relerr(y, want) < 8e-3
    assert _relerr(x.grad, xf.grad) < 1.5e-2
    assert _relerr(lin.lora_A.weight.grad, Af.grad) < 1.5e-2
    assert _relerr(lin.lora_B.weight.grad, Bf.grad) < 1.5e-2
    # eval: no dropout
    lin.eval()
    with torch.no_grad():
        ye = lin(x)
    wante = ref.lora_linear(xf.detach(), lin.weight.float(), None, Af.detach(), Bf.detach(), lin.scaling)
    assert _relerr(ye, wante) < 8e-3


def test_merge_kernel_matches_reference():
    from relora_b200.ops import reference as ref
    from relora_b200.relora import ReLoRaLinear

    torch.manual_seed(0)
    lin = ReLoRaLinear(768, 2560, r=128, lora_alpha=32, bias=False).cuda().to(BF)
    lin.weight.data.normal_(std=0.02)
    lin.lora_B.weight.data.normal_(std=0.02)
    want = ref.merge_delta(lin.weight.data, lin.lora_A.weight.data, lin.lora_B.weight.data, lin.scaling)
    from relora_b200.ops import fused

    assert fused.merge_and_reinit_modules([lin], seed=1, restart_index=2)
    assert _relerr(lin.weight.data, want) < 3e-3
    assert float(lin.lora_B.weight.abs().sum()) == 0
    assert float(lin.lora_A.weight.float().abs().max()) <= 1 / math.sqrt(768) + 1e-4


def test_llama_module_path_on_gpu_matches_cpu_reference():
    """llama_9m-sized model: fused leaf ops on the GPU vs the PyTorch path (same weights)."""
    import os

    from relora_b200.models import LlamaForCausalLM, load_config
    from relora_b200.ops import dispatch
    from relora_b200.relora import ReLoRaModel

    cfg = load_config(os.path.join(os.path.dirname(os.path.dirname(__file__)), "configs", "llama_20m.json"))
    torch.manual_seed(0)
    m = LlamaForCausalLM(cfg)
    w = ReLoRaModel(m, r=64, lora_alpha=32, lora_dropout=0.0, target_modules=["attn", "mlp"], init_lora_a="kaiming")
    for mod in w.relora_modules():
        torch.nn.init.normal_(mod.lora_B.weight, std=0.02)
    w = w.cuda().to(BF)
    ids = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda")
    w.train()
    loss = w(input_ids=ids, labels=ids).loss
    loss.backward()
    g_fused = {n: p.grad.float().clone() for n, p in w.named_parameters() if p.grad is not None}
    w.zero_grad(set_to_none=True)
    dispatch.force_reference(True)
    try:
        loss_ref = w(input_ids=ids, labels=ids).loss
        loss_ref.backward()
    finally:
        dispatch.force_reference(False)
    assert abs(float(loss) - float(loss_ref)) < 3e-2
    for n, p in w.named_parameters():
        if p.grad is not None and ("lora_B" in n or "embed" in n):
            assert _relerr(g_fused[n], p.grad.float()) < 0.12, n


# ----------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("B,T,nh,hd", [(2, 512, 4, 48), (1, 320, 2, 64), (3, 128, 2, 32), (1, 1000, 3, 64), (2, 64, 1, 16)])
def test_attention_fwd_bwd(C, B, T, nh, hd):
    """wgmma causal flash attention over the packed qkv buffer vs an fp32 PyTorch reference (forward, lse and dq/dk/dv)."""
    torch.manual_seed(T + hd)
    h = nh * hd
    qkv = _rand(B * T, 3 * h)
    out = torch.zeros(B * T, h, device="cuda", dtype=BF)
    lse = torch.zeros(B, nh, T, device="cuda", dtype=torch.float32)
    scale = 1.0 / math.sqrt(hd)
    C.attention_fwd(qkv, out, lse, B, T, nh, hd, scale)
    q, k, v = (qkv.view(B, T, 3, nh, hd)[:, :, i].transpose(1, 2).float().detach().requires_grad_() for i in range(3))
    s = (q @ k.transpose(-1, -2)) * scale
    mask = torch.ones(T, T, dtype=torch.bool, device="cuda").tril()
    s = s.masked_fill(~mask, float("-inf"))
    p = torch.softmax(s, dim=-1)
    want = p @ v  # [B, nh, T, hd]
    got = out.view(B, T, nh, hd).transpose(1, 2)
    assert _relerr(got, want) < 8e-3
    want_lse = torch.logsumexp(s, dim=-1) / math.log(2.0)
    assert (lse - want_lse).abs().max() < 2e-2
    dout = _rand(B * T, h, scale=0.5)
    want.backward(dout.view(B, T, nh, hd).transpose(1, 2).float())
    delta = torch.empty(B, nh, T, device="cuda", dtype=torch.float32)
    # both backward forms: dQ recomputing S / dP, and dQ = dS·K from the dSᵀ tiles the dK/dV kernel stores (the default)
    for use_ws in (False, True):
        dqkv = torch.zeros(B * T, 3 * h, device="cuda", dtype=BF)
        ws = torch.full((C.attention_ds_workspace_elems(B, T, nh),), float("nan"), device="cuda", dtype=BF) if use_ws else None
        C.attention_bwd(qkv, out, dout, lse, delta, dqkv, B, T, nh, hd, scale, ws)
        d5 = dqkv.view(B, T, 3, nh, hd)
        for i, (name, ref_t) in enumerate((("dq", q), ("dk", k), ("dv", v))):
            e = _relerr(d5[:, :, i].transpose(1, 2), ref_t.grad)
            assert e < 2e-2, (name, use_ws, e)


# ----------------------------------------------------------------------------------------- fp8 frozen-weight path
@pytest.mark.parametrize("M,N,K,pair", [(256, 256, 256, 0), (1000, 768, 640, 0), (512, 1024, 2048, 1), (12288, 2304, 768, 0)])
def test_gemm_fp8_frozen_path_with_bf16_lora_branch(C, F, M, N, K, pair):
    """x·Wᵀ on the E4M3 tensor-core path (e4m3 wgmma, per-tensor scales) with the bf16 LoRA branch accumulated into
    the same register accumulator; checked against an fp32 product of the *dequantised* operands."""
    torch.manual_seed(K + N)
    r = 128
    x, W = _rand(M, K), _rand(N, K, scale=0.05)
    u, B = _rand(M, r), _rand(N, r, scale=0.05)
    res = _rand(M, N)
    f32 = lambda v: torch.tensor([v], dtype=torch.float32, device="cuda")  # noqa: E731
    scratch, sw, inv_sw = f32(0.0), f32(0.0), f32(0.0)
    W8 = torch.empty(N, K, dtype=torch.uint8, device="cuda")
    C.fp8_quantize_weight(W, W8, scratch, sw, inv_sw)
    assert abs(float(sw) - float(W.float().abs().max()) / 448.0) < 1e-6
    sx = float(x.float().abs().max()) / 448.0
    x8 = torch.empty(M, K, dtype=torch.uint8, device="cuda")
    amax = f32(0.0)
    C.fp8_quantize_act(x, x8, f32(1.0 / sx), amax)
    assert abs(float(amax) - float(x.float().abs().max())) < 1e-6
    xq = x8.view(torch.float8_e4m3fn).float() * sx
    Wq = W8.view(torch.float8_e4m3fn).float() * float(sw)
    assert _relerr(xq, x) < 0.05 and _relerr(Wq, W) < 0.05  # E4M3: 3 mantissa bits
    alpha = sx * float(sw)
    u_scaled = (u.float() / alpha).to(BF)  # the LoRA term shares the accumulator, so it is pre-divided by the product scale
    out = torch.empty(M, N, device="cuda", dtype=BF)
    F.gemm(x8, W8, out, M=M, N=N, K1=K, a2=u_scaled, b2=B, K2=r, residual=res, fp8=True, alpha_dev=f32(alpha),
           block_n=256 if pair else 0, pair=pair)
    want = xq @ Wq.t() + (u_scaled.float() * alpha) @ B.float().t() + res.float()
    assert _relerr(out, want) < 6e-3
    # and it is close to the unquantised product (quantisation noise only)
    full = x.float() @ W.float().t() + u.float() @ B.float().t() + res.float()
    assert _relerr(out, full) < 0.06


def test_producers_emit_the_same_e4m3_copy_as_the_standalone_quantiser(C):
    """RMSNorm / SwiGLU / dropout_expand can write the E4M3 copy of their output themselves (fp8 frozen-weight path):
    bit-identical to quantising the bf16 output afterwards, same recorded amax."""
    torch.manual_seed(0)
    f32 = lambda v: torch.tensor([v], dtype=torch.float32, device="cuda")  # noqa: E731
    M, H, Fd = 300, 768, 2560
    seed = torch.tensor([31], dtype=torch.int32, device="cuda")
    inv = f32(448.0 / 6.0)

    def ref_q(y):
        q, am = torch.empty(y.shape, dtype=torch.uint8, device="cuda"), f32(0.0)
        C.fp8_quantize_act(y, q, inv, am)
        return q, float(am)

    # RMSNorm (+ 2 dropout copies)
    x, w = _rand(M, H), (1.0 + 0.1 * torch.randn(H, device="cuda")).to(BF)
    y, rstd = torch.empty_like(x), torch.empty(M, device="cuda", dtype=torch.float32)
    xd = torch.empty(M, 2 * H, device="cuda", dtype=BF)
    q, am = torch.empty(M, H, dtype=torch.uint8, device="cuda"), f32(0.0)
    C.rmsnorm_fwd(x, w, y, rstd, 1e-6, xd, seed, [1, 2], 0.1, q, inv, am)
    rq, ram = ref_q(y)
    assert torch.equal(q, rq) and float(am) == ram
    # SwiGLU (+ dropout copy)
    gu = _rand(M, 2 * Fd)
    h, hd = torch.empty(M, Fd, device="cuda", dtype=BF), torch.empty(M, Fd, device="cuda", dtype=BF)
    q, am = torch.empty(M, Fd, dtype=torch.uint8, device="cuda"), f32(0.0)
    C.swiglu_fwd(gu, h, hd, seed, 5, 0.1, q, inv, am)
    rq, ram = ref_q(h)
    assert torch.equal(q, rq) and float(am) == ram
    # dropout_expand: E4M3 copy of the un-dropped input
    a = _rand(M, H)
    ad = torch.empty(M, H, device="cuda", dtype=BF)
    q, am = torch.empty(M, H, dtype=torch.uint8, device="cuda"), f32(0.0)
    C.dropout_expand(a, ad, seed, [7], 0.1, q, inv, am)
    rq, ram = ref_q(a)
    assert torch.equal(q, rq) and float(am) == ram


# ----------------------------------------------------------------------------------------- GPT-NeoX / Pythia leaf kernels
@pytest.mark.parametrize("M,H,bias", [(300, 512, True), (257, 2048, True), (64, 768, False), (33, 1000, True)])
def test_layernorm_fwd_bwd(F, M, H, bias):
    torch.manual_seed(0)
    x = (torch.randn(M, H, device="cuda") * 2 + 0.5).to(BF).requires_grad_()
    w = (1 + 0.1 * torch.randn(H, device="cuda")).to(BF).requires_grad_()
    b = (0.1 * torch.randn(H, device="cuda")).to(BF).requires_grad_() if bias else None
    dy = _rand(M, H)
    y = F.layernorm(x, w, b, 1e-5)
    y.backward(dy)
    xf, wf = x.detach().float().requires_grad_(), w.detach().float().requires_grad_()
    bf = b.detach().float().requires_grad_() if bias else None
    yf = torch.nn.functional.layer_norm(xf, (H,), wf, bf, 1e-5)
    yf.backward(dy.float())
    assert _relerr(y, yf) < 6e-3
    assert _relerr(x.grad, xf.grad) < 8e-3 and _relerr(w.grad, wf.grad) < 8e-3
    if bias:
        assert _relerr(b.grad, bf.grad) < 8e-3


@pytest.mark.parametrize("tanh_approx", [False, True])
def test_gelu_fwd_bwd(F, tanh_approx):
    torch.manual_seed(0)
    z = (torch.randn(777, 264, device="cuda") * 2).to(BF).requires_grad_()
    da = _rand(777, 264)
    a = F.gelu(z, tanh_approx)
    a.backward(da)
    zf = z.detach().float().requires_grad_()
    af = torch.nn.functional.gelu(zf, approximate="tanh" if tanh_approx else "none")
    af.backward(da.float())
    assert _relerr(a, af) < 5e-3 and _relerr(z.grad, zf.grad) < 6e-3


@pytest.mark.parametrize("nh,hd,rot", [(8, 64, 16), (4, 128, 32), (2, 256, 64)])
def test_neox_partial_rope(F, nh, hd, rot):
    """In-place partial rotary on the fused query_key_value layout vs the reference expression (modeling_pythia.py:172-197)."""
    from relora_b200.models.pythia import GPTNeoXRotaryEmbedding, apply_partial_rotary

    torch.manual_seed(0)
    B, T = 2, 37
    qkv = _rand(B, T, nh, 3 * hd).requires_grad_()
    rope = GPTNeoXRotaryEmbedding(rot, 128, device="cuda")
    cos, sin = rope(qkv, seq_len=T)
    out = F.neox_rope(qkv, cos[0, 0].float().contiguous(), sin[0, 0].float().contiguous(), nh, hd, rot)
    g = _rand(B, T, nh, 3 * hd)
    out.backward(g)
    ref_in = qkv.detach().float().requires_grad_()
    q = ref_in[..., :hd].permute(0, 2, 1, 3)
    k = ref_in[..., hd:2 * hd].permute(0, 2, 1, 3)
    pos = torch.arange(T, device="cuda").unsqueeze(0).expand(B, T)
    qr, kr = apply_partial_rotary(q[..., :rot], k[..., :rot], cos.float(), sin.float(), pos)
    qf = torch.cat((qr, q[..., rot:]), -1).permute(0, 2, 1, 3)
    kf = torch.cat((kr, k[..., rot:]), -1).permute(0, 2, 1, 3)
    want = torch.cat((qf, kf, ref_in[..., 2 * hd:]), -1)
    want.backward(g.float())
    assert _relerr(out, want) < 5e-3 and _relerr(qkv.grad, ref_in.grad) < 5e-3


def test_pythia_native_leaf_ops_match_eager():
    """Tiny Pythia on CUDA/bf16: LayerNorm / GELU / partial rotary / (head 64) attention kernels vs the same model forced onto the
    PyTorch expressions (RELORA_B200_FORCE_REFERENCE semantics through ops.dispatch.force_reference)."""
    from relora_b200.models import GPTNeoXForCausalLM, SimpleConfig
    from relora_b200.ops import dispatch

    torch.manual_seed(0)
    cfg = SimpleConfig(model_type="gpt_neox", vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                       intermediate_size=1024, rotary_pct=0.25, max_position_embeddings=128, layer_norm_eps=1e-5,
                       use_parallel_residual=True, hidden_act="gelu", rotary_emb_base=10000, tie_word_embeddings=False)
    model = GPTNeoXForCausalLM(cfg).to("cuda", BF).train()
    ids = torch.randint(0, 512, (2, 64), device="cuda")
    out = model(input_ids=ids, labels=ids)
    out.loss.backward()
    g_native = {n: p.grad.float().clone() for n, p in model.named_parameters()}
    model.zero_grad()
    dispatch.force_reference(True)
    try:
        ref = model(input_ids=ids, labels=ids)
        ref.loss.backward()
    finally:
        dispatch.force_reference(False)
    assert abs(float(out.loss) - float(ref.loss)) < 3e-2
    worst = max(_relerr(g_native[n], p.grad) for n, p in model.named_parameters() if p.grad is not None and float(p.grad.float().norm()) > 0)
    assert worst < 0.08, worst


def test_module_path_attention_uses_the_wgmma_kernels(F):
    """`F.causal_attention` (module path) vs torch SDPA on q, k, v [B, nh, T, hd] incl. the gradients."""
    torch.manual_seed(0)
    B, nh, T, hd = 2, 4, 200, 48
    q, k, v = (_rand(B, nh, T, hd).requires_grad_() for _ in range(3))
    do = _rand(B, nh, T, hd)
    o = F.causal_attention(q, k, v)
    o.backward(do)
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    of = torch.nn.functional.scaled_dot_product_attention(qf, kf, vf, is_causal=True)
    of.backward(do.float())
    assert _relerr(o, of) < 1e-2
    for a, b in ((q.grad, qf.grad), (k.grad, kf.grad), (v.grad, vf.grad)):
        assert _relerr(a, b) < 2e-2


# ----------------------------------------------------------------------------------------- block-scaled MXFP8 (csrc/gemm_mx.cu)
def test_mx_quantisers_match_the_oracle(C):
    from relora_b200.ops import mx

    torch.manual_seed(0)
    x = _rand(200, 328, scale=3.0)
    x[5] = 0                      # an all-zero row: scale 2^-127, zeros
    q, sf = mx.quantize_rows(x)
    assert q.shape == (200, 384)
    # dequantise through the weight path to check values: quantise the same matrix as a "weight" with 1 x 32 semantics is not
    # available, so compare through a GEMM with the identity instead (see test_mx_gemm); here: bytes of the padding are zero
    assert int(q[:, 328:].max()) == 0
    w = _rand(264, 328, scale=0.05)
    mw = mx.quantize_weight(w)
    deq = mx.dequantize_weight(mw).float()
    ref = mx.ref_quantize_weight_2d(w)
    # the scale exponent may differ by one where amax / 448 sits on a power of two (log2f rounding): compare values, not bytes
    assert _relerr(deq, ref) < 2e-2 and _relerr(deq, w) < 4e-2
    # merge: W += delta, requantised in place
    delta = torch.randn(264, 328, device="cuda") * 0.01
    mx.merge_(mw, delta)
    assert _relerr(mx.dequantize_weight(mw), mx.ref_quantize_weight_2d(deq + delta)) < 2e-2


@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (384, 256, 512), (300, 264, 328), (1024, 768, 768)])
def test_mx_gemm_forward_and_input_gradient(C, M, N, K):
    """e4m3 wgmma per 32-element scale block vs the fp32 product of the dequantised operands."""
    from relora_b200.ops import mx

    torch.manual_seed(1)
    x = _rand(M, K, scale=1.5)
    w = _rand(N, K, scale=0.03)
    mw = mx.quantize_weight(w)
    wd = mx.dequantize_weight(mw).float()
    y = mx.linear(x, mw)
    want = mx.ref_quantize_rows(x) @ wd.t()
    assert _relerr(y, want) < 1e-2, ("forward", _relerr(y, want))
    # input gradient: the same bytes read MN-major, reduction over N
    dy = _rand(M, N, scale=0.7)
    xr = x.clone().requires_grad_()
    mx.linear(xr, mw).backward(dy)
    want_dx = mx.ref_quantize_rows(dy) @ wd
    assert _relerr(xr.grad, want_dx) < 1e-2, ("dx", _relerr(xr.grad, want_dx))
    # LoRA segment in the same accumulator + residual
    u, B = _rand(M, 128, scale=0.5), _rand(N, 128, scale=0.05)
    res = _rand(M, N)
    out = torch.empty(M, N, device="cuda", dtype=BF)
    xq, sfx = mx.quantize_rows(x)
    C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, out, M, N, K, False, u, B, res)
    want2 = want + u.float() @ B.float().t() + res.float()
    assert _relerr(out, want2) < 1e-2


def test_mx_relora_linear_packed_storage_trains():
    """`ReLoRaLinear(quantize="mxfp8")` on CUDA: packed-only storage (0.53x of bf16), block-scaled tensor-core forward / dx, merge."""
    from relora_b200.relora import ReLoRaLinear
    from relora_b200.utils import frozen_weight_bytes

    torch.manual_seed(0)
    w = torch.randn(512, 768) * 0.02
    lin = ReLoRaLinear(768, 512, r=128, lora_alpha=32, bias=False, weight_data=w.clone(), quantize="mxfp8", lora_dropout=0.0).to("cuda", BF)
    b = frozen_weight_bytes(torch.nn.Sequential(lin))
    assert b["resident_bytes"] / b["bf16_bytes"] < 0.54
    torch.nn.init.normal_(lin.lora_B.weight, std=0.02)
    x = _rand(256, 768).requires_grad_()
    y = lin(x)
    y.float().pow(2).mean().backward()
    wd = lin.weight.float()
    want = x.detach().float() @ wd.t() + (x.detach().float() @ lin.lora_A.weight.float().t() @ lin.lora_B.weight.float().t()) * lin.scaling
    assert _relerr(y, want) < 3e-2
    assert x.grad is not None and bool(torch.isfinite(x.grad).all()) and lin.lora_A.weight.grad is not None
    before = wd.clone()
    target = before + float(lin.scaling) * lin.lora_B.weight.float() @ lin.lora_A.weight.float()
    lin.merge_and_reinit()
    assert _relerr(lin.weight.float(), target) < 4e-2 and float(lin.lora_B.weight.abs().sum()) == 0
