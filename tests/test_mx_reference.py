"""The exact contract of the block-scaled MXFP8 path (ops/reference.py, block-scaled MXFP8 section) on the CPU: the scale layout
against the formula of csrc/gemm_mx.cu, the exponent rule against a brute-force search, the encoding against torch's E4M3
conversion, gemm_mx_ref against the product of the decoded operands, and assert_gemm_close rejecting each single scale or edge
error at the shapes the GPU sweep (test_mx_modes_gpu.py) uses."""
import math

import numpy as np
import pytest
import torch

from relora_b200.ops import quant
from relora_b200.ops import reference as ref

BF, F64 = torch.bfloat16, torch.float64


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def block_scaled(rows, cols, gen, tile_rows):
    """bf16 ``[rows, cols]`` whose every block of ``tile_rows`` x 32 has its own power-of-two magnitude: neighbours in either
    direction differ (exponent (i + 2j) mod 5 - 2 for block (i, j))."""
    i = torch.arange(rows).unsqueeze(1) // tile_rows
    j = torch.arange(cols).unsqueeze(0) // 32
    return (torch.randn(rows, cols, generator=gen) * torch.exp2(((i + 2 * j) % 5 - 2).double()).float()).to(BF)


# ----------------------------------------------------------------------------------------------- scale layout
def test_sf_offset_is_the_layout_of_the_kernel_header():
    """byte[(r % 32)·16 + (r / 32)·4 + j] of the 512-byte block [row block][k group], and every scale of an operand has its
    own byte of the mx_sf_bytes array."""
    for rows, k in ((1, 8), (127, 328), (300, 768), (129, 32)):
        kg = (k + 127) // 128
        for row in range((rows + 127) // 128 * 128):
            for col in range(kg * 4):
                rb, r, g, j = row // 128, row % 128, col // 4, col % 4
                assert ref.mx_sf_offset(row, col, kg) == (rb * kg + g) * 512 + (r % 32) * 16 + (r // 32) * 4 + j
        idx = ref._sf_index(rows, k).reshape(-1)
        assert idx.numel() == ref.mx_sf_bytes(rows, k)
        assert torch.equal(idx.sort().values, torch.arange(ref.mx_sf_bytes(rows, k)))
        grid = torch.randint(0, 256, ((rows + 127) // 128 * 128, kg * 4), generator=_gen(rows + k), dtype=torch.uint8)
        assert torch.equal(ref.mx_scale_grid(ref.mx_scale_pack(grid, rows, k), rows, k), grid)


# ----------------------------------------------------------------------------------------------- exponent rule
def _brute_exponent(a: float) -> int:
    for e in range(-127, 128):
        if a <= 448.0 * 2.0 ** e:
            return e
    return 127


def _f32_neighbours(x):
    x32 = np.float32(x)
    return [float(np.nextafter(x32, np.float32(-np.inf))), float(x32), float(np.nextafter(x32, np.float32(np.inf)))]


def _bf16_neighbours(x):
    b = torch.tensor([x], dtype=torch.float32).to(BF).view(torch.int16)
    return [float(torch.tensor([int(b) + d], dtype=torch.int16).view(BF).float()) for d in (-1, 0, 1)]


def test_scale_exponent_is_exact_at_every_boundary():
    """448·2^e exactly and its fp32 / bf16 neighbours either side for every e a finite fp32 amax can take, zero, fp32 and bf16
    subnormals, the clamp at -127 and the largest finite values."""
    vals = [0.0, 2.0 ** -149, 2.0 ** -133, 2.0 ** -127, 2.0 ** -126, 448.0 * 2.0 ** -127, 1.0, float(np.finfo(np.float32).max),
            float(torch.finfo(BF).max)]
    for e in range(-127, 121):
        b = 448.0 * 2.0 ** e
        if b <= float(np.finfo(np.float32).max):
            vals += _f32_neighbours(b) + _bf16_neighbours(b)
    vals = [v for v in vals if math.isfinite(v) and v >= 0]
    got = ref.mx_scale_exponent(torch.tensor(vals, dtype=F64))
    want = torch.tensor([_brute_exponent(v) for v in vals])
    bad = (got != want).nonzero()
    assert bad.numel() == 0, [(vals[int(i)], int(got[i]), int(want[i])) for i in bad[:5, 0]]
    assert int(ref.mx_scale_exponent(torch.tensor([0.0], dtype=F64))) == -127
    assert int(ref.mx_scale_exponent(torch.tensor([448.0], dtype=F64))) == 0
    assert int(ref.mx_scale_exponent(torch.tensor([float(np.nextafter(np.float32(448), np.float32(1e9)))], dtype=F64))) == 1


def test_log2_rule_disagrees_where_the_exact_rule_is_needed():
    """The rounded ceil(log2(amax / 448)) of the earlier PyTorch quantisers (fp32 amax, as in a merged weight) gives a
    different exponent than the exact rule at some fp32 neighbours of 448·2^e."""
    vals = []
    for e in range(-120, 120):
        vals += _f32_neighbours(448.0 * 2.0 ** e)
    a = torch.tensor(vals, dtype=torch.float32)
    old = torch.ceil(torch.log2(a / 448.0)).clamp(-127, 127).to(torch.int64)
    exact = ref.mx_scale_exponent(a.double())
    assert torch.equal(exact, torch.tensor([_brute_exponent(v) for v in vals]))
    assert bool((old != exact).any()), "the fp32 log2 form agrees everywhere here"


# ----------------------------------------------------------------------------------------------- encoding
def _expected_block(x64):
    """Independent per-block encoding with Python floats: (bytes, scale byte)."""
    finite = [abs(v) for v in x64 if not math.isnan(v)]
    amax = max(finite, default=0.0)
    if math.isinf(amax):
        q = torch.tensor([v * 0.0 for v in x64], dtype=torch.float32)
        return q.to(torch.float8_e4m3fn).view(torch.uint8), 0xFF
    e = _brute_exponent(amax)
    q = torch.tensor([v * 2.0 ** -e for v in x64], dtype=F64).float().clamp(-448, 448)
    return q.to(torch.float8_e4m3fn).view(torch.uint8), e + 127


def test_encoding_matches_the_float8_conversion():
    g = _gen(3)
    blocks = (torch.randn(64, 32, generator=g) * torch.exp2(torch.randint(-30, 30, (64, 1), generator=g).float())).to(BF).double()
    for i, e in enumerate(range(-20, 20, 2)):  # the block maximum exactly on 448·2^e and on its bf16 neighbours
        for j, v in enumerate(_bf16_neighbours(448.0 * 2.0 ** e)):
            blocks[3 * i + j, 5] = -v if j == 1 else v
    blocks[60] = 0.0
    blocks[61] = torch.tensor(_bf16_neighbours(2.0 ** -130) * 10 + [0.0, 2.0 ** -133], dtype=F64)  # bf16 subnormals only
    blocks[62, 7] = float("nan")
    blocks[63, 3] = float("-inf")
    blocks[59] = float("nan")
    q, s = ref.mx_encode_blocks(blocks)
    for r in range(blocks.shape[0]):
        want_q, want_s = _expected_block(blocks[r].tolist())
        assert int(s[r]) == want_s, (r, int(s[r]), want_s)
        ref.assert_e4m3_bytes_equal(f"block {r}", q[r], want_q)
    assert int(s[60]) == 0 and int(s[59]) == 0 and int(s[63]) == ref.MX_SF_NAN
    assert int(s[61]) == 0 and bool((q[61, :20] != 0).any())  # subnormal inputs are encoded at 2^127, not flushed
    assert (int(q[62, 7]) & 0x7F) == 0x7F and int(s[62]) == int(ref.mx_encode_blocks(blocks[62:63].nan_to_num(0.0))[1])
    assert (int(q[63, 3]) & 0x7F) == 0x7F and bool((q[63, :3] & 0x7F == 0).all())


def test_quantize_rows_exact_pads_and_round_trips():
    g = _gen(4)
    for M, K in ((1, 8), (127, 328), (129, 32), (300, 768)):
        x = block_scaled(M, K, g, 1)
        q, sf = ref.mx_quantize_rows_exact(x)
        Kp = (K + 127) // 128 * 128
        assert q.shape == (M, Kp) and sf.numel() == ref.mx_sf_bytes(M, K)
        assert int(q[:, K:].abs().sum()) == 0
        grid = ref.mx_scale_grid(sf, M, K)
        assert int(grid[M:].sum()) == 0 and int(grid[:, (K + 31) // 32:].sum()) == 0  # padding rows / blocks: zero blocks
        d = ref.mx_decode_rows(q, sf, M, K)
        x64 = x.double()
        assert bool(((d - x64).abs() <= x64.abs() * 2.0 ** -4 + 2.0 ** -9 * torch.exp2(grid[:M].double() - 127).repeat_interleave(
            32, 1)[:, :K]).all())
        # the CPU layout (ops/quant.py) encodes the same 1 x 32 blocks identically
        qw = quant.quantize(x, "mxfp8")
        Kb = (K + 31) // 32
        assert torch.equal(qw.scales, grid[:M, :Kb])
        assert torch.equal(qw.data, q[:, :Kb * 32])


def test_weight_2d_exact_scale_layouts_and_merge():
    g = _gen(5)
    N, K = 300, 328
    w = block_scaled(N, K, g, 32)
    q, sf_fwd, sf_bwd = ref.mx_quantize_weight_2d_exact(w)
    Np, Kp = 384, 384
    assert q.shape == (Np, Kp) and int(q[N:].abs().sum()) == 0 and int(q[:, K:].abs().sum()) == 0
    fwd, bwd = ref.mx_scale_grid(sf_fwd, N, K), ref.mx_scale_grid(sf_bwd, K, N)
    tiles = fwd[::32]  # [Np/32, Kp/32]
    assert torch.equal(fwd, tiles.repeat_interleave(32, 0)) and torch.equal(bwd, tiles.t().repeat_interleave(32, 0))
    assert len(set(tiles[:9, :10].reshape(-1).tolist())) > 3  # tiles carry distinct scales
    # merge: a zero delta keeps every value; a delta is added in fp32 to the decoded weight and requantised
    q0, f0, b0 = ref.mx_quantize_weight_2d_exact(q_old=q, sf_old=sf_fwd, delta=torch.zeros(N, K), N=N, K=K)
    assert torch.equal(ref.mx_decode_weight(q0, f0, N, K), ref.mx_decode_weight(q, sf_fwd, N, K))
    delta = torch.randn(N, K, generator=g) * 0.01
    q1, f1, b1 = ref.mx_quantize_weight_2d_exact(q_old=q, sf_old=sf_fwd, delta=delta)
    v = (ref.mx_decode_weight(q, sf_fwd, N, K).float() + delta).to(F64)
    d1 = ref.mx_decode_weight(q1, f1, N, K)
    s1 = torch.exp2(ref.mx_scale_grid(f1, N, K)[:N].double() - 127).repeat_interleave(32, 1)[:, :K]
    assert bool(((d1 - v).abs() <= v.abs() * 2.0 ** -4 + 2.0 ** -9 * s1).all())
    # an Inf in one tile of the delta: that tile's scale is 0xFF and it decodes non-finite, nothing else changes
    delta[40, 70] = float("inf")
    q3, f3, b3 = ref.mx_quantize_weight_2d_exact(q_old=q, sf_old=sf_fwd, delta=delta)
    t = ref.mx_scale_grid(f3, N, K)[::32]
    assert int(t[1, 2]) == ref.MX_SF_NAN and int((t == ref.MX_SF_NAN).sum()) == 1
    d3 = ref.mx_decode_weight(q3, f3, N, K)
    tile = torch.zeros(N, K, dtype=torch.bool)
    tile[32:64, 64:96] = True
    assert not bool(torch.isfinite(d3[tile]).any()) and torch.equal(d3[~tile], d1[~tile])


# ----------------------------------------------------------------------------------------------- gemm_mx_ref
def _operands(M, N, K, seed):
    """Forward (x·Wᵀ, B K-major) and input-gradient (dy·W, B MN-major) operands built by the exact quantisers."""
    g = _gen(seed)
    x, dy, w = block_scaled(M, K, g, 1), block_scaled(M, N, g, 1), block_scaled(N, K, g, 32)
    xq, sfx = ref.mx_quantize_rows_exact(x)
    dq, sfd = ref.mx_quantize_rows_exact(dy)
    wq, sf_fwd, sf_bwd = ref.mx_quantize_weight_2d_exact(w)
    return dict(x=(xq, sfx), dy=(dq, sfd), w=(wq, sf_fwd, sf_bwd), g=g)


def test_gemm_mx_ref_is_the_product_of_the_decoded_operands():
    M, N, K = 300, 264, 328
    o = _operands(M, N, K, 6)
    (xq, sfx), (dq, sfd), (wq, sf_fwd, sf_bwd) = o["x"], o["dy"], o["w"]
    X, DY = ref.mx_decode_rows(xq, sfx, M, K), ref.mx_decode_rows(dq, sfd, M, N)
    W = ref.mx_decode_weight(wq, sf_fwd, N, K)
    Wt = ref.mx_decode_weight(wq.t().contiguous(), sf_bwd, K, N)  # the backward layout reads the transposed tiles
    assert torch.equal(Wt, W.t())
    got, bound = ref.gemm_mx_ref(xq, sfx, wq, sf_fwd, M, N, K)
    torch.testing.assert_close(got, X @ W.t(), rtol=1e-12, atol=0)
    torch.testing.assert_close(bound, X.abs() @ W.abs().t(), rtol=1e-12, atol=0)
    got, _ = ref.gemm_mx_ref(dq, sfd, wq, sf_bwd, M, K, N, b_mn_major=True)
    torch.testing.assert_close(got, DY @ W, rtol=1e-12, atol=0)
    a2, b2 = torch.randn(M, 64, generator=o["g"]).to(BF), torch.randn(N, 64, generator=o["g"]).to(BF)
    res = torch.randn(M, N, generator=o["g"]).to(BF)
    got, bound = ref.gemm_mx_ref(xq, sfx, wq, sf_fwd, M, N, K, a2=a2, b2=b2, residual=res)
    want = X @ W.t() + a2.double() @ b2.double().t() + res.double()
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    assert bool((bound >= got.abs() - 1e-9).all())


# ----------------------------------------------------------------------------------------------- sensitivity
M_S, N_S, K_S = 300, 264, 328  # ragged M and N, a partial last k-block; Np = Kp = 384 (a square 12 x 12 tile grid)


def _regrid(sf, rows, k, fn):
    return ref.mx_scale_pack(fn(ref.mx_scale_grid(sf, rows, k).clone()), rows, k)


def _mutation(name):
    """(output of a kernel with one scale or edge error, exact reference, bound)."""
    o = _operands(M_S, N_S, K_S, 7)
    (xq, sfx), (dq, sfd), (wq, sf_fwd, sf_bwd) = o["x"], o["dy"], o["w"]
    fwd = dict(a=xq, sfa=sfx, b=wq, sfb=sf_fwd, M=M_S, N=N_S, K=K_S)
    bwd = dict(a=dq, sfa=sfd, b=wq, sfb=sf_bwd, M=M_S, N=K_S, K=N_S, b_mn_major=True)
    if name in ("residual_row", "last_mtile_row"):
        res = torch.randn(M_S, N_S, generator=o["g"]).to(BF)
        want, bound = ref.gemm_mx_ref(**fwd, residual=res)
        bad = want.clone()
        if name == "residual_row":
            bad[200] -= res[200].double()
        else:  # the last row of the last (partial) M tile is never stored
            bad[M_S - 1] = 0.0
        return bad, want, bound
    call = bwd if name in ("sf_fwd_for_sf_bwd", "tile_scale_transposed") else fwd
    want, bound = ref.gemm_mx_ref(**call)
    mut = dict(call)
    if name == "row_group_neighbour":  # rows 32..63 of x read the scales of rows 0..31
        mut["sfa"] = _regrid(sfx, M_S, K_S, lambda gr: torch.cat([gr[:32], gr[:32], gr[64:]]))
    elif name == "kcol_off_by_one":  # the weight scale of k-block j + 1 used for k-block j
        mut["sfb"] = _regrid(sf_fwd, N_S, K_S, lambda gr: torch.cat([gr[:, 1:], gr[:, -1:]], 1))
    elif name == "sf_fwd_for_sf_bwd":
        mut["sfb"] = sf_fwd
    elif name == "tile_scale_transposed":  # the backward array filled with tile (k/32, n/32) instead of (n/32, k/32)
        mut["sfb"] = _regrid(sf_bwd, K_S, N_S, lambda gr: gr[::32].t().repeat_interleave(32, 0))
    elif name == "last_kblock_dropped":  # K = 328: the partial k-block (columns 320..327) skipped
        a = xq.clone()
        a[:, 320:] = 0
        mut["a"] = a
    else:
        raise ValueError(name)
    bad, _ = ref.gemm_mx_ref(**mut)
    return bad, want, bound


MUTATIONS = ["row_group_neighbour", "kcol_off_by_one", "sf_fwd_for_sf_bwd", "tile_scale_transposed", "last_kblock_dropped",
             "last_mtile_row", "residual_row"]


@pytest.mark.parametrize("name", MUTATIONS)
def test_assert_gemm_close_rejects_one_scale_or_edge_error(name):
    bad, want, bound = _mutation(name)
    assert bool(torch.isfinite(want).all())
    assert ref.assert_gemm_close(want.to(BF), want, bound, fp8=True) <= 1.0  # the exact result, rounded, passes
    with pytest.raises(AssertionError):
        ref.assert_gemm_close(bad.to(BF), want, bound, fp8=True)
