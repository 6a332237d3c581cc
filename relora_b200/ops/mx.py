"""Block-scaled MXFP8 storage + compute for the frozen weights (``--quantize 8bit`` / ``mxfp8`` on CUDA): Python face of
``csrc/gemm_mx.cu``.

* :class:`MxWeight` — the ONLY resident form of a frozen weight: E4M3 bytes ``[Npad, Kpad]`` (padded to multiples of 128) plus one
  UE8M0 scale per 32 x 32 tile, expanded into the two scale-factor arrays the tensor core reads (forward: reduction over ``K``;
  input gradient: reduction over ``N``, same bytes read MN-major).  1.06 bytes per parameter instead of 2.
* :func:`linear` — autograd function ``y = x · Wᵀ (+ bias)``: activations are quantised per (row, 32 columns) on the fly, both GEMMs run
  e4m3 ``wgmma`` per 32-element block with the scale factors applied to the fp32 partial products.
* :func:`merge_` — the ReLoRA merge on packed storage: dequantise → fp32 add → requantise with fresh tile scales, in place
  (reference ``relora.py:277-299``).

The pure-PyTorch functions at the bottom are the numerics oracle (tests/test_kernels_gpu.py).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch

from . import native

__all__ = ["MxWeight", "quantize_weight", "dequantize_weight", "quantize_rows", "linear", "merge_", "supported",
           "ref_quantize_rows", "ref_quantize_weight_2d"]

_BF16 = torch.bfloat16


def _pad128(n: int) -> int:
    return (n + 127) // 128 * 128


def supported(n: int, k: int) -> bool:
    """Shapes the kernels take: reduction / output widths that are multiples of 8 (TMA pitch, vector accesses)."""
    return n % 8 == 0 and k % 8 == 0


@dataclass
class MxWeight:
    q: torch.Tensor        # uint8 [Npad, Kpad] E4M3 bytes (zero padding)
    sf_fwd: torch.Tensor   # uint8, scale of (row n, 32-block of k) in the blocked layout of csrc/gemm_mx.cu
    sf_bwd: torch.Tensor   # uint8, scale of (row k, 32-block of n)
    N: int
    K: int

    @property
    def nbytes(self) -> int:
        return int(self.q.numel() + self.sf_fwd.numel() + self.sf_bwd.numel())

    def to(self, device) -> "MxWeight":
        return MxWeight(self.q.to(device), self.sf_fwd.to(device), self.sf_bwd.to(device), self.N, self.K)


def _alloc(N: int, K: int, device) -> MxWeight:
    C = native.require()
    return MxWeight(torch.zeros(_pad128(N), _pad128(K), dtype=torch.uint8, device=device),
                    torch.zeros(C.mx_sf_bytes(N, K), dtype=torch.uint8, device=device),
                    torch.zeros(C.mx_sf_bytes(K, N), dtype=torch.uint8, device=device), N, K)


@torch.no_grad()
def quantize_weight(w: torch.Tensor) -> MxWeight:
    N, K = w.shape
    mw = _alloc(N, K, w.device)
    native.require().mx_quantize_weight_2d(w.to(_BF16).contiguous(), None, mw.q, mw.sf_fwd, mw.sf_bwd, N, K)
    return mw


@torch.no_grad()
def dequantize_weight(mw: MxWeight, dtype=_BF16) -> torch.Tensor:
    out = torch.empty(mw.N, mw.K, dtype=_BF16, device=mw.q.device)
    native.require().mx_dequantize_weight(mw.q, mw.sf_fwd, out)
    return out if dtype == _BF16 else out.to(dtype)


@torch.no_grad()
def merge_(mw: MxWeight, delta: torch.Tensor) -> None:
    """``W += delta`` on the packed weight: dequantise, add in fp32, requantise every 32 x 32 tile with a fresh scale (in place)."""
    native.require().mx_quantize_weight_2d(None, delta.to(torch.float32).contiguous(), mw.q, mw.sf_fwd, mw.sf_bwd, mw.N, mw.K)


@torch.no_grad()
def quantize_rows(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``x`` bf16 ``[M, K]`` → (E4M3 bytes ``[M, Kpad]``, scale factors per (row, 32 columns))."""
    C = native.require()
    M, K = x.shape
    q = torch.empty(M, _pad128(K), dtype=torch.uint8, device=x.device)
    sf = torch.empty(C.mx_sf_bytes(M, K), dtype=torch.uint8, device=x.device)
    C.mx_quantize_rows(x.contiguous(), q, sf)
    return q, sf


class _MxLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mw: MxWeight, a2, b2):
        C = native.require()
        shp = x.shape
        x2 = x.reshape(-1, shp[-1]).to(_BF16).contiguous()
        M = x2.shape[0]
        xq, sfx = quantize_rows(x2)
        y = torch.empty(M, mw.N, dtype=_BF16, device=x.device)
        C.gemm_mx(xq, sfx, mw.q, mw.sf_fwd, y, M, mw.N, mw.K, False, a2, b2, None)
        ctx.mw = mw
        ctx.shape = shp
        ctx.lora = (a2, b2)
        return y.view(*shp[:-1], mw.N)

    @staticmethod
    def backward(ctx, dy):
        C = native.require()
        mw = ctx.mw
        dy2 = dy.reshape(-1, mw.N).to(_BF16).contiguous()
        M = dy2.shape[0]
        dq, sfd = quantize_rows(dy2)
        dx = torch.empty(M, mw.K, dtype=_BF16, device=dy.device)
        # dx = dy · W: the same E4M3 bytes read MN-major, reduction over N with the backward scale array
        C.gemm_mx(dq, sfd, mw.q, mw.sf_bwd, dx, M, mw.K, mw.N, True, None, None, None)
        return dx.view(ctx.shape), None, None, None


def linear(x: torch.Tensor, mw: MxWeight, bias: Optional[torch.Tensor] = None, a2: Optional[torch.Tensor] = None,
           b2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``y = x · Wᵀ (+ a2 · b2ᵀ in the same accumulator) (+ bias)`` with ``W`` block-scaled E4M3.  ``a2 [.., r]`` / ``b2 [N, r]`` (bf16,
    no gradient through this call) are the LoRA up-projection operands of the fused executor."""
    y = _MxLinearFn.apply(x, mw, a2, b2)
    return y if bias is None else y + bias


# ----------------------------------------------------------------------------- PyTorch oracle
def _ue8m0(amax: torch.Tensor) -> torch.Tensor:
    e = torch.ceil(torch.log2(torch.clamp(amax, min=2.0 ** -127) / 448.0)).clamp(-127, 127)
    return torch.exp2(e)


def ref_quantize_rows(x: torch.Tensor) -> torch.Tensor:
    """Dequantised value of the row-wise (1 x 32) MXFP8 quantisation of ``x`` (fp32)."""
    M, K = x.shape
    Kp = (K + 31) // 32 * 32
    xf = torch.nn.functional.pad(x.float(), (0, Kp - K)).view(M, Kp // 32, 32)
    s = _ue8m0(xf.abs().amax(-1, keepdim=True))
    q = (xf / s).clamp(-448, 448).to(torch.float8_e4m3fn).float()
    return (q * s).view(M, Kp)[:, :K]


def ref_quantize_weight_2d(w: torch.Tensor) -> torch.Tensor:
    """Dequantised value of the 32 x 32-tile MXFP8 quantisation of ``w`` (fp32)."""
    N, K = w.shape
    Np, Kp = (N + 31) // 32 * 32, (K + 31) // 32 * 32
    wf = torch.nn.functional.pad(w.float(), (0, Kp - K, 0, Np - N)).view(Np // 32, 32, Kp // 32, 32)
    s = _ue8m0(wf.abs().amax(dim=(1, 3), keepdim=True))
    q = (wf / s).clamp(-448, 448).to(torch.float8_e4m3fn).float()
    return (q * s).view(Np, Kp)[:N, :K]
