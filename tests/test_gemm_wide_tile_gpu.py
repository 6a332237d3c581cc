"""The 192-wide output tile of the wgmma GEMM and of the LoRA input-gradient kernel gives the bits of the 128-wide tile.

A tile's width does not change the order in which an output element sums over K, and the epilogue's fp32 operations are
the same at both widths (the residual short path included), so every call form the executors issue must agree bit for
bit.  M 12416 runs 97 M tiles; M 328 ends inside a tile, so its last tile takes the general epilogue.  Operands sit inside
NaN-guarded buffers and outputs inside sentinel-guarded ones (guarded_buffers.py)."""
import pytest
import torch

from guarded_buffers import Guarded

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
R = 128
SENTINEL = 1234.0


@pytest.fixture(scope="module")
def F():
    from relora_b200.ops import fused

    fused._C()
    return fused


def _rand(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(BF)


def _operand(t):
    return Guarded(t, float("nan")).view


def _run(call, shape):
    o = Guarded(torch.empty(*shape, dtype=BF, device="cuda"), SENTINEL, interior=torch.full(shape, float("nan"), dtype=BF, device="cuda"))
    call(o.view)
    torch.cuda.synchronize()
    assert o.guards_intact(), "the output guard region was written"
    got = o.view.clone()
    assert not torch.isnan(got).any(), "an output element was not written"
    return got


def _same_bits(F, a1, b1, M, N, **kw):
    ops = {k: (_operand(v) if torch.is_tensor(v) else v) for k, v in kw.items()}
    A1, B1 = _operand(a1), _operand(b1)
    got = {bn: _run(lambda out: F.gemm(A1, B1, out, M=M, N=N, block_n=bn, pair=0, **ops), (M, N)) for bn in (128, 192)}
    assert torch.equal(got[128], got[192]), f"192-wide differs from 128-wide in {int((got[128] != got[192]).sum())} elements"


@pytest.mark.parametrize("M", [328, 12416])
@pytest.mark.parametrize("N", [768, 704])  # 704: the last tile holds two of its three 64-column sub-tiles
def test_plain_and_residual(F, M, N):
    torch.manual_seed(M + N)
    K = 768
    x, W = _rand(M, K), _rand(N, K, scale=0.05)
    _same_bits(F, x, W, M, N, K1=K)
    _same_bits(F, x, W, M, N, K1=K, residual=_rand(M, N))


@pytest.mark.parametrize("M", [328, 12416])
def test_grouped_qkv_with_lora(F, M):
    torch.manual_seed(M)
    K, Ng, G = 768, 768, 3
    x, W, u, B = _rand(M, K), _rand(G * Ng, K, scale=0.05), _rand(M, G * R), _rand(G * Ng, R, scale=0.05)
    _same_bits(F, x, W, M, G * Ng, K1=K, a2=u, b2=B, K2=R, n_per_group=Ng, a2_group_kofs=R)


@pytest.mark.parametrize("M", [328, 12416])
def test_mn_major_input_gradient_base(F, M):
    torch.manual_seed(M + 1)
    N, K = 768, 5120
    dy, W = _rand(M, K), _rand(K, N, scale=0.05)  # W [K, N] read MN-major: the gate / up input gradient's base product
    _same_bits(F, dy, W, M, N, K1=K, b1_mn=True)


@pytest.mark.parametrize("M", [328, 12416])
def test_ragged_group(F, M):
    """groups of 2560 columns: each group's last 192-wide tile stores one 64-column sub-tile"""
    torch.manual_seed(M + 2)
    K, Ng, G = 768, 2560, 2
    x, W, u, B = _rand(M, K), _rand(G * Ng, K, scale=0.05), _rand(M, G * R), _rand(G * Ng, R, scale=0.05)
    _same_bits(F, x, W, M, G * Ng, K1=K, a2=u, b2=B, K2=R, n_per_group=Ng, a2_group_kofs=R)


@pytest.mark.parametrize("with_base", [False, True])
@pytest.mark.parametrize("G", [1, 2, 3])
@pytest.mark.parametrize("M", [328, 12416])
def test_lora_dx(F, M, G, with_base):
    """dropout p = 0.1; two or three groups run on the 128-wide tile whatever the request, so they must agree too"""
    C = F._C()
    torch.manual_seed(G * 100 + M)
    N, Ng = 768, 768
    dy, W = _operand(_rand(M, G * Ng)), _operand(_rand(G * Ng, N, scale=0.05))
    du, A = _operand(_rand(M, G * R)), _operand(_rand(G * R, N, scale=0.05))
    base = _operand(_rand(M, N))
    seed = torch.tensor([1234567], dtype=torch.int32, device="cuda")
    keys = [11, 22, 33][:G]

    def call(bn):
        if with_base:
            return lambda out: C.lora_dx(None, None, du, A, out, seed, keys, 0.1, base, pair=0, block_n=bn)
        return lambda out: C.lora_dx(dy, W, du, A, out, seed, keys, 0.1, pair=0, block_n=bn)

    got = {bn: _run(call(bn), (M, N)) for bn in (128, 192)}
    assert torch.equal(got[128], got[192]), f"192-wide differs from 128-wide in {int((got[128] != got[192]).sum())} elements"
