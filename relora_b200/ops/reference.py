"""Plain PyTorch definitions of every fused operator (the numerics oracle + the CPU path).

Each function states the exact math the sm_90a kernel of the same name implements; GPU tests
compare kernel output against these evaluated in fp32.  Reference sites are cited per op.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------- dropout mask
# Counter-based keep-mask shared bit-for-bit by the CUDA kernels (csrc/common.cuh: keep_drop()).
# h = lowbias32(row*C1 ^ (col>>1)*C2 ^ seed);  keep(row, col) = ((col & 1) ? h >> 16 : h & 0xFFFF) >= round(p * 2^16)
_C1 = 0x9E3779B1
_C2 = 0x85EBCA77
_M32 = 0xFFFFFFFF


def _lowbias32(x: torch.Tensor) -> torch.Tensor:
    x = x & _M32
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & _M32
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & _M32
    x = x ^ (x >> 16)
    return x


def dropout_threshold(p: float) -> int:
    """16-bit keep threshold (see :func:`dropout_keep_mask`)."""
    return int(round(p * (1 << 16)))


def dropout_keep_mask(seed: int, rows: int, cols: int, p: float, device=None, row_offset: int = 0, col_offset: int = 0) -> torch.Tensor:
    """Boolean ``[rows, cols]`` keep mask for dropout probability ``p`` and 32-bit ``seed``."""
    r = torch.arange(row_offset, row_offset + rows, dtype=torch.int64, device=device).unsqueeze(1)
    c = torch.arange(col_offset, col_offset + cols, dtype=torch.int64, device=device).unsqueeze(0)
    # one 32-bit hash per column pair, its halves compared against a 16-bit threshold (csrc/common.cuh:keep_drop)
    x = ((r * _C1) & _M32) ^ (((c >> 1) * _C2) & _M32) ^ (int(seed) & _M32)
    h = _lowbias32(x)
    half = torch.where((c & 1) == 1, h >> 16, h & 0xFFFF)
    return half >= dropout_threshold(p)


def random_prune_keep_mask(seed: int, n: int, ratio: float, device=None, offset: int = 0) -> torch.Tensor:
    """Keep mask of the hash-based random pruning of ``n`` consecutive elements starting at flat index ``offset``
    (one 24-bit draw per element; ``csrc/optim.cu:random_prune_kernel`` / ``common.cuh:keep_bit``)."""
    c = torch.arange(offset, offset + n, dtype=torch.int64, device=device)
    x = ((c * _C2) & _M32) ^ (int(seed) & _M32)
    return (_lowbias32(x) >> 8) >= int(round(ratio * (1 << 24)))


def mix_seed(base: int, *keys: int) -> int:
    """Derive a 32-bit stream seed from a base seed and integer keys (step, module id, ...)."""
    x = int(base) & _M32
    for k in keys:
        x = (x ^ (int(k) & _M32)) & _M32
        x = ((x ^ (x >> 16)) * 0x7FEB352D) & _M32
        x = ((x ^ (x >> 15)) * 0x846CA68B) & _M32
        x = x ^ (x >> 16)
    return x


# ----------------------------------------------------------------------------- norms
def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    """fp32 normalise -> round to weight dtype -> scale (reference modeling_llama.py:83-91)."""
    var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    y = (x.to(torch.float32) * torch.rsqrt(var + eps)).to(weight.dtype)
    return weight * y


def rmsnorm_fp32(x, weight, eps):
    """All-fp32 variant used as the tolerance anchor for kernel tests."""
    xf = x.to(torch.float32)
    return xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * weight.to(torch.float32)


# ----------------------------------------------------------------------------- rotary
def rope_tables(head_dim: int, n_pos: int, base: float = 10000.0, device=None, dtype=torch.float32) -> Tuple[torch.Tensor, torch.Tensor]:
    inv = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.float32, device=device) / head_dim))
    f = torch.outer(torch.arange(n_pos, dtype=torch.float32, device=device), inv)
    emb = torch.cat((f, f), -1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rope_apply(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """``x``: [..., T, hd]; ``cos``/``sin``: [T, hd] (half-rotation layout)."""
    h = x.shape[-1] // 2
    rot = torch.cat((-x[..., h:], x[..., :h]), -1)
    return x * cos + rot * sin


# ----------------------------------------------------------------------------- LoRA linear
def lora_linear(
    x: torch.Tensor,
    weight: Optional[torch.Tensor],
    bias: Optional[torch.Tensor],
    lora_a: torch.Tensor,
    lora_b: torch.Tensor,
    scale: float,
    *,
    p: float = 0.0,
    seed: Optional[int] = None,
    residual: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """y = x Wᵀ + b + s·((m ⊙ x)/(1-p)) Aᵀ Bᵀ (+ residual), all accumulated in fp32.

    ``m`` is :func:`dropout_keep_mask` over the flattened ``[tokens, in]`` view (reference
    ``relora.py:309-323`` with ``nn.Dropout`` replaced by the counter-based mask).
    """
    shp = x.shape
    x2 = x.reshape(-1, shp[-1]).to(torch.float32)
    xd = x2
    if p > 0.0:
        assert seed is not None
        keep = dropout_keep_mask(seed, x2.shape[0], x2.shape[1], p, device=x.device)
        xd = x2 * keep / (1.0 - p)
    u = xd @ lora_a.to(torch.float32).t()
    y = (u @ lora_b.to(torch.float32).t()) * scale
    if weight is not None:
        y = y + x2 @ weight.to(torch.float32).t()
    if bias is not None:
        y = y + bias.to(torch.float32)
    if residual is not None:
        y = y + residual.reshape(-1, y.shape[-1]).to(torch.float32)
    return y.reshape(*shp[:-1], y.shape[-1])


def swiglu(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    """silu(gate) * up (reference modeling_llama.py:157-158)."""
    return F.silu(gate.to(torch.float32)) * up.to(torch.float32)


# ----------------------------------------------------------------------------- LM head + CE
def lm_head_cross_entropy(h: torch.Tensor, w_head: torch.Tensor, labels: torch.Tensor, chunk: int = 4096, ignore_index: int = -100) -> torch.Tensor:
    """Mean next-token cross-entropy without materialising ``[B, T, V]`` logits.

    Equivalent to ``CrossEntropyLoss()(logits[:, :-1], labels[:, 1:])`` with
    ``logits = h @ w_headᵀ`` (reference modeling_llama.py:692-708); computed chunk by chunk in fp32.
    """
    B, T, H = h.shape
    hs = h[:, :-1].reshape(-1, H)
    tgt = labels[:, 1:].reshape(-1).to(h.device)
    total = torch.zeros((), dtype=torch.float32, device=h.device)
    count = torch.zeros((), dtype=torch.float32, device=h.device)
    for s in range(0, hs.shape[0], chunk):
        logits = (hs[s : s + chunk] @ w_head.t()).to(torch.float32)
        t = tgt[s : s + chunk]
        total = total + F.cross_entropy(logits, t, reduction="sum", ignore_index=ignore_index)
        count = count + (t != ignore_index).sum()
    return total / count.clamp(min=1)


# ----------------------------------------------------------------------------- optimizer
def adamw_step(
    param: torch.Tensor,
    grad: torch.Tensor,
    exp_avg: torch.Tensor,
    exp_avg_sq: torch.Tensor,
    *,
    step: int,
    lr: float,
    beta1: float,
    beta2: float,
    eps: float,
    weight_decay: float,
    grad_scale: float = 1.0,
) -> None:
    """One decoupled-weight-decay Adam step, fp32 math, results rounded to the storage dtypes
    (``torch.optim.AdamW`` semantics, reference torchrun_main.py:666; ``grad_scale`` folds the
    1/(world·accum) average and the clip coefficient)."""
    g = grad.to(torch.float32) * grad_scale
    p = param.to(torch.float32)
    m = exp_avg.to(torch.float32)
    v = exp_avg_sq.to(torch.float32)
    p = p * (1.0 - lr * weight_decay)
    m = beta1 * m + (1.0 - beta1) * g
    v = beta2 * v + (1.0 - beta2) * g * g
    bc1 = 1.0 - beta1**step
    bc2 = 1.0 - beta2**step
    denom = v.sqrt() / math.sqrt(bc2) + eps
    p = p - (lr / bc1) * (m / denom)
    param.copy_(p.to(param.dtype))
    exp_avg.copy_(m.to(exp_avg.dtype))
    exp_avg_sq.copy_(v.to(exp_avg_sq.dtype))


# ----------------------------------------------------------------------------- merge
def merge_delta(weight: torch.Tensor, lora_a: torch.Tensor, lora_b: torch.Tensor, scale: float) -> torch.Tensor:
    """W + s·B@A accumulated in fp32, rounded to ``weight.dtype`` (reference relora.py:275-276)."""
    return (weight.to(torch.float32) + scale * (lora_b.to(torch.float32) @ lora_a.to(torch.float32))).to(weight.dtype)


def kaiming_uniform_from_hash(seed: int, rows: int, cols: int, bound: float, device=None) -> torch.Tensor:
    """U(-bound, bound) from the same counter hash the merge kernel uses: 24 random bits per element."""
    r = torch.arange(rows, dtype=torch.int64, device=device).unsqueeze(1)
    c = torch.arange(cols, dtype=torch.int64, device=device).unsqueeze(0)
    x = ((r * _C1) & _M32) ^ ((c * _C2) & _M32) ^ (int(seed) & _M32)
    u = (_lowbias32(x) >> 8).to(torch.float32) * (1.0 / (1 << 24))  # [0, 1)
    return (2.0 * u - 1.0) * bound
