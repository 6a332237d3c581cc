"""Block-scaled MXFP8 storage + compute for the frozen weights (``--quantize 8bit`` / ``mxfp8`` on CUDA): Python face of
``csrc/gemm_mx.cu``.

* :class:`MxWeight` — the ONLY resident form of a frozen weight: E4M3 bytes ``[Npad, Kpad]`` (padded to multiples of 128) plus one
  UE8M0 scale per 32 x 32 tile, expanded into the two scale-factor arrays the tensor core reads (forward: reduction over ``K``;
  input gradient: reduction over ``N``, same bytes read MN-major).  1.06 bytes per parameter instead of 2.
* :func:`linear` — autograd function ``y = x · Wᵀ (+ bias)``: activations are quantised per (row, 32 columns) on the fly, both GEMMs run
  e4m3 ``wgmma`` per 32-element block with the scale factors applied to the fp32 partial products.
* :func:`merge_` — the ReLoRA merge on packed storage: dequantise → fp32 add → requantise with fresh tile scales, in place
  (reference ``relora.py:277-299``).

The pure-PyTorch functions at the bottom decode the exact contracts of ops/reference.py (block-scaled MXFP8 section).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch

from . import native, reference

__all__ = ["MxWeight", "quantize_weight", "dequantize_weight", "quantize_rows", "linear", "merge_", "supported",
           "sf_blocks", "stack_weights", "stack_part", "refresh_part", "ref_quantize_rows", "ref_quantize_weight_2d"]

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


# ----------------------------------------------------------------------------- stacked weights (the fused executor)
# A stack is the row concatenation of packed weights that share K, each part starting on a 128-row boundary (its Npad rows).
# Its q and forward scale array are the parts' bytes one after another, so a part is a slice of them.  The input-gradient scale
# array is not: its 512-byte blocks are ordered [128-row block of K][128-group of N], so a part's blocks are a strided window of
# the stack's, and a part keeps a copy of its own.
def sf_blocks(sf: torch.Tensor, rows: int, k: int) -> torch.Tensor:
    """The scale array of a ``[rows, k]`` operand as its ``[pad128(rows)/128, pad128(k)/128, 512]`` blocks."""
    return sf.view(_pad128(rows) // 128, _pad128(k) // 128, 512)


def stack_weights(parts) -> MxWeight:
    """The stack of packed weights ``parts`` (one K): byte for byte what quantising the stacked matrix gives, since every
    32 x 32 tile lies inside one part."""
    K = parts[0].K
    assert all(p.K == K for p in parts)
    q = torch.cat([p.q for p in parts])
    N = q.shape[0]
    sf_fwd = torch.cat([p.sf_fwd for p in parts])
    sf_bwd = torch.cat([sf_blocks(p.sf_bwd, K, p.N) for p in parts], dim=1).reshape(-1)
    return MxWeight(q, sf_fwd, sf_bwd, N, K)


def stack_part(stack: MxWeight, r0: int, N: int) -> MxWeight:
    """The packed weight of rows ``[r0, r0 + N)`` of ``stack`` (``r0`` a multiple of 128): q and the forward scales alias the
    stack, the input-gradient scales are a copy (:func:`refresh_part`)."""
    kg = _pad128(stack.K) // 128
    o = r0 // 128 * kg * 512
    part = MxWeight(stack.q[r0:r0 + _pad128(N)], stack.sf_fwd[o:o + _pad128(N) // 128 * kg * 512],
                    torch.empty(reference.mx_sf_bytes(stack.K, N), dtype=torch.uint8, device=stack.q.device), N, stack.K)
    refresh_part(stack, part, r0)
    return part


def refresh_part(stack: MxWeight, part: MxWeight, r0: int) -> None:
    """Copy the input-gradient scales of ``part`` (rows ``[r0, ...)`` of ``stack``) out of the stack's."""
    g0 = r0 // 128
    sf_blocks(part.sf_bwd, part.K, part.N).copy_(sf_blocks(stack.sf_bwd, stack.K, stack.N)[:, g0:g0 + _pad128(part.N) // 128])


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
def ref_quantize_rows(x: torch.Tensor) -> torch.Tensor:
    """Dequantised value of the row-wise (1 x 32) MXFP8 quantisation of ``x`` (fp32; the exact contract of
    :func:`quantize_rows`, ops/reference.py)."""
    q, sf = reference.mx_quantize_rows_exact(x.to(_BF16))
    return reference.mx_decode_rows(q, sf, *x.shape).float()


def ref_quantize_weight_2d(w: torch.Tensor) -> torch.Tensor:
    """Dequantised value of the 32 x 32-tile MXFP8 quantisation of ``w`` (fp32; the exact contract of :func:`quantize_weight`,
    ops/reference.py)."""
    N, K = w.shape
    q, sf_fwd, _ = reference.mx_quantize_weight_2d_exact(w.to(_BF16))
    return reference.mx_decode_weight(q, sf_fwd, N, K).float()
