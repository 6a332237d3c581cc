"""Plain PyTorch definitions of every fused operator (the numerics oracle + the CPU path).

Each function states the exact math the sm_90a kernel of the same name implements; GPU tests
compare kernel output against these evaluated in fp32.  Reference sites are cited per op.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import numpy as np
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


# ----------------------------------------------------------------------------- wgmma GEMM (csrc/gemm.h)
# fp64 evaluations of the GemmDesc / LoraDxDesc contracts, written from their documentation.  Each returns the exact result and
# an element-wise magnitude bound (sum of |terms|) that scales the accumulation-error tolerance of assert_gemm_close.
_F64 = torch.float64

# Accumulation-error coefficients of assert_gemm_close, as a fraction of the element's magnitude bound.  Set from the worst
# element observed on an H100 80GB HBM3 (sm_90a wgmma) over the mode sweep in tests/test_gemm_modes_gpu.py, with headroom:
# |err| / bound of fp32 outputs reached 2.0e-7 for bf16 operands (split-K atomics included) and 3.2e-4 for fp8 operands, whose
# tensor-core path accumulates with fewer mantissa bits.
GEMM_C_ACC_BF16 = 2.0 ** -16
GEMM_C_ACC_FP8 = 2.0 ** -10


def _window(t: torch.Tensor, r0: int, nr: int, c0: int, nc: int, what: str) -> torch.Tensor:
    """``t[r0:r0+nr, c0:c0+nc]``; a window that leaves the operand is an error, not a silent truncation."""
    if r0 < 0 or c0 < 0 or r0 + nr > t.shape[0] or c0 + nc > t.shape[1]:
        raise IndexError(f"{what}: window rows [{r0}, {r0 + nr}) x cols [{c0}, {c0 + nc}) outside the {tuple(t.shape)} operand")
    return t[r0:r0 + nr, c0:c0 + nc]


def _gemm_operand(t: torch.Tensor, mn_major: bool, fp8_dtype=None) -> torch.Tensor:
    """fp64 ``[rows, K]`` view of an operand: K-major element (i, k) is ``t[i, k]``, MN-major it is ``t[k, i]``."""
    if fp8_dtype is not None:
        t = t.view(fp8_dtype)
    t = t.to(_F64)
    return t.t() if mn_major else t


def gemm_ref(
    a1: torch.Tensor,
    b1: torch.Tensor,
    out: Optional[torch.Tensor] = None,
    *,
    M: Optional[int] = None,
    N: Optional[int] = None,
    K1: Optional[int] = None,
    a2: Optional[torch.Tensor] = None,
    b2: Optional[torch.Tensor] = None,
    K2: int = 0,
    a1_mn: bool = False,
    b1_mn: bool = False,
    n_per_group: int = 0,
    a1_group_kofs: int = 0,
    a2_group_kofs: int = 0,
    residual: Optional[torch.Tensor] = None,
    alpha: float = 1.0,
    accumulate: bool = False,
    out_dtype: torch.dtype = torch.bfloat16,
    block_n: int = 0,
    split_k: int = 1,
    b1_group_kofs: int = 0,
    b1_local_n: bool = False,
    m_per_group: int = 0,
    b1_mn_ofs_per_mgroup: int = 0,
    bias: Optional[torch.Tensor] = None,
    pair: int = -1,
    fp8: int = 0,
    alpha_dev: Optional[torch.Tensor] = None,
) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp64 ``(result, bound)`` of :func:`relora_b200.ops.fused.gemm` called with the same arguments (``out``: its content
    before the call; read only when ``accumulate`` is set, otherwise only its dtype matters).

    Per output element (m, n), with n in column group g = n // n_per_group and local column nl = n - g·n_per_group:

        D = alpha·alpha_dev · ( Σ_k A1[m, g·a1_group_kofs + k] · B1[j, g·b1_group_kofs + k]      (k < K1)
                              + Σ_k A2[m, g·a2_group_kofs + k] · B2[n, k] )                    (k < K2)
        j = (nl if b1_local_n else n) + (m // m_per_group) · b1_mn_ofs_per_mgroup

    bf16 output: out = D + bias[n] + residual[m, n] (+ out if accumulate), rounded once; fp32 output: out = D (+ out).
    ``fp8``: A1 / B1 are one-byte tensors decoded as E4M3 (A1 as E5M2 with ``fp8=2``).  ``block_n``, ``split_k`` and
    ``pair`` choose the schedule and do not change the result.  ``bound`` is the same sum over |terms|."""
    if M is None:
        M = a1.shape[1] if a1_mn else a1.shape[0]
    if K1 is None:
        K1 = a1.shape[0] if a1_mn else a1.shape[1]
    if N is None:
        N = b1.shape[1] if b1_mn else b1.shape[0]
    if a2 is not None and K2 == 0:
        K2 = b2.shape[1]
    odt = out.dtype if out is not None else out_dtype
    if odt == torch.float32 and (bias is not None or residual is not None):
        raise ValueError("gemm: bias and residual are only fused for bf16 outputs")
    if accumulate and out is None:
        raise ValueError("gemm: accumulate needs the previous output")
    f8a = (torch.float8_e5m2 if fp8 == 2 else torch.float8_e4m3fn) if fp8 else None
    A1 = _gemm_operand(a1, a1_mn, f8a)
    B1 = _gemm_operand(b1, b1_mn, torch.float8_e4m3fn if fp8 else None)
    A2 = _gemm_operand(a2, False) if K2 > 0 else None
    B2 = _gemm_operand(b2, False) if K2 > 0 else None
    npg = n_per_group if n_per_group > 0 else N
    mpg = m_per_group if m_per_group > 0 else M
    ref = torch.zeros(M, N, dtype=_F64, device=a1.device)
    bound = torch.zeros_like(ref)
    for g in range((N + npg - 1) // npg):
        n0, nw = g * npg, min(npg, N - g * npg)
        for m0 in range(0, M, mpg):
            mw = min(mpg, M - m0)
            j0 = (0 if b1_local_n else n0) + (m0 // mpg) * b1_mn_ofs_per_mgroup
            a = _window(A1, m0, mw, g * a1_group_kofs, K1, "A1")
            b = _window(B1, j0, nw, g * b1_group_kofs, K1, "B1")
            ref[m0:m0 + mw, n0:n0 + nw] += a @ b.t()
            bound[m0:m0 + mw, n0:n0 + nw] += a.abs() @ b.abs().t()
        if K2 > 0:
            a = _window(A2, 0, M, g * a2_group_kofs, K2, "A2")
            b = _window(B2, n0, nw, 0, K2, "B2")
            ref[:, n0:n0 + nw] += a @ b.t()
            bound[:, n0:n0 + nw] += a.abs() @ b.abs().t()
    scale = float(alpha) * (float(alpha_dev.reshape(-1)[0]) if alpha_dev is not None else 1.0)
    ref *= scale
    bound *= abs(scale)
    for extra in (None if bias is None else bias.reshape(-1)[:N].to(_F64).expand(M, N),
                  None if residual is None else residual[:M, :N].to(_F64),
                  out[:M, :N].to(_F64) if accumulate else None):
        if extra is not None:
            ref += extra
            bound += extra.abs()
    return ref, bound


def lora_dx_ref(dy, w, du: torch.Tensor, a: torch.Tensor, seed, keys, p: float, base: Optional[torch.Tensor] = None):
    """fp64 ``(result, bound)`` of the extension's ``lora_dx(dy, w, du, a, out, seed, keys, p, base)``:

        out = dy·W + 1/(1-p) · Σ_g keep_g ⊙ (du_g·A_g),    keep_g = dropout_keep_mask(mix_seed(seed, keys[g]), M, N, p)

    with ``du = [du_0 | du_1 | ...]`` ([M, G·r]) and ``A = [A_0; A_1; ...]`` ([G·r, N]); with ``base`` given (the ``Kb == 0``
    form) ``base`` replaces dy·W.  ``seed``: the device seed tensor or an int (None reads as 0)."""
    G = len(keys)
    M, N = du.shape[0], a.shape[1]
    r = du.shape[1] // G
    s = 0 if seed is None else (int(seed.reshape(-1)[0].item()) if torch.is_tensor(seed) else int(seed)) & _M32
    ref = torch.zeros(M, N, dtype=_F64, device=du.device)
    bound = torch.zeros_like(ref)
    for g in range(G):
        x, y = du[:, g * r:(g + 1) * r].to(_F64), a[g * r:(g + 1) * r].to(_F64)
        part, pb = x @ y, x.abs() @ y.abs()
        if p > 0:
            keep = dropout_keep_mask(mix_seed(s, keys[g]), M, N, p, device=du.device)
            part, pb = part * keep, pb * keep
        ref += part
        bound += pb
    inv_keep = 1.0 / (1.0 - p)
    ref *= inv_keep
    bound *= inv_keep
    if base is not None:
        ref += base[:M, :N].to(_F64)
        bound += base[:M, :N].to(_F64).abs()
    else:
        x, y = dy.to(_F64), w.to(_F64)
        ref += x @ y
        bound += x.abs() @ y.abs()
    return ref, bound


def assert_gemm_close(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, *, fp8: bool = False) -> float:
    """Element-wise check of a GEMM output against :func:`gemm_ref` / :func:`lora_dx_ref`:

        |out - ref| <= c_out·|ref| + c_acc·bound

    ``c_out`` is the output rounding (2⁻⁸ for bf16, 2⁻²³ for fp32), ``c_acc`` the accumulation error per unit of the
    magnitude bound (:data:`GEMM_C_ACC_BF16`, or :data:`GEMM_C_ACC_FP8` for the fp8 tensor-core path).  A NaN fails.
    Returns the worst ratio of error to tolerance (<= 1 when it passes); the failure message names where it occurs."""
    M, N = ref.shape
    o = out[:M, :N].to(_F64)
    c_out = 2.0 ** -8 if out.dtype == torch.bfloat16 else 2.0 ** -23
    c_acc = GEMM_C_ACC_FP8 if fp8 else GEMM_C_ACC_BF16
    err = (o - ref).abs()
    tol = c_out * ref.abs() + c_acc * bound
    ratio = torch.where(tol > 0, err / tol.clamp(min=1e-300), torch.where(err == 0, 0.0, math.inf))
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
    flat = int(torch.argmax(ratio))
    i, j = divmod(flat, N)
    worst = float(ratio[i, j])
    if not worst <= 1.0:
        n_bad = int((ratio > 1.0).sum())
        raise AssertionError(
            f"GEMM output out of tolerance at {n_bad} of {M * N} elements; worst ratio {worst:.3g} at (row {i}, col {j}): "
            f"out={float(o[i, j]):.6g} ref={float(ref[i, j]):.6g} bound={float(bound[i, j]):.6g} (c_out={c_out:.3g}, c_acc={c_acc:.3g})")
    return worst


# ----------------------------------------------------------------------------- wgmma attention (csrc/attention.h)
# Coefficients of assert_attention_close.  ATTN_C_P / ATTN_C_D are analytic: bf16 round-to-nearest has a unit roundoff of 2⁻⁸
# (8 significant bits), and P (forward, dV) and dS (dQ, dK) are packed to bf16 once as wgmma register operands; twice that
# rounding leaves room for the fp32 accumulation, ex2.approx and the fp32 row sums, which are all below 2⁻²⁰ relative.
# ATTN_C_S / ATTN_C_L are set from the worst element observed on an H100 80GB HBM3 (700 W) over tests/test_attention_modes_gpu.py,
# with headroom: the lse error reached 1.0e-7·(1 + |lse|) where the score term is zero (q = 0), and 5.0e-7 per unit of the score
# term elsewhere (the rising-maximum regime at head_dim 128, the c_l share included).  ATTN_C_S is the constant the GEMM uses for
# the same fp32 wgmma accumulation (GEMM_C_ACC_BF16).
ATTN_C_P = 2.0 ** -7
ATTN_C_D = 2.0 ** -7
ATTN_C_S = 2.0 ** -16
ATTN_C_L = 2.0 ** -20
# The kernels flush fp32 subnormals (ex2.approx.ftz, FTZ arithmetic): every term of a sum may lose up to this much absolutely.
ATTN_FTZ = 2.0 ** -126
_ATTN_C = {"out": ATTN_C_P, "lse": ATTN_C_L, "dq": ATTN_C_D, "dk": ATTN_C_D, "dv": ATTN_C_D}
_LOG2E = 1.0 / math.log(2.0)


def attention_unpack(x: torch.Tensor, B: int, T: int, nh: int, hd: int, *, nkv: int = -1, interleaved: bool = False):
    """Views ``(q, k, v)`` — ``[B, nh, T, hd]``, ``[B, nkv, T, hd]``, ``[B, nkv, T, hd]`` — of a packed ``qkv`` / ``dqkv``
    buffer ``[B*T, (nh + 2·nkv)·hd]``: ``[q: nh | k: nkv | v: nkv]`` heads per row, or ``[nh, (q|k|v), hd]`` when
    ``interleaved`` (GPT-NeoX ``query_key_value``).  A ``[B*T, nh·hd]`` buffer (``out`` / ``dout``) unpacks with
    :func:`attention_heads`."""
    nkv = nh if nkv < 0 else nkv
    if interleaved and nkv != nh:
        raise ValueError("attention: the interleaved layout has no grouped-query form")
    if interleaved:
        x5 = x.reshape(B, T, nh, 3, hd)
        return tuple(x5[:, :, :, i].transpose(1, 2) for i in range(3))
    x4 = x.reshape(B, T, nh + 2 * nkv, hd)
    return tuple(x4[:, :, a:b].transpose(1, 2) for a, b in ((0, nh), (nh, nh + nkv), (nh + nkv, nh + 2 * nkv)))


def attention_heads(x: torch.Tensor, B: int, T: int, nh: int, hd: int) -> torch.Tensor:
    """``[B, nh, T, hd]`` view of a ``[B*T, nh·hd]`` buffer (``out`` / ``dout``)."""
    return x.reshape(B, T, nh, hd).transpose(1, 2)


def _spread(w: torch.Tensor, v: torch.Tensor, o: torch.Tensor) -> torch.Tensor:
    """Σ_k w_ik |v_kj − o_ij| over ``w [B, H, T, T]``, ``v, o [B, H, T, hd]``, a few query rows at a time."""
    Bh, T, hd = w.shape[0] * w.shape[1], w.shape[2], v.shape[-1]
    res = torch.empty_like(o)
    step = max(1, (1 << 24) // (Bh * T * hd))
    for i0 in range(0, T, step):
        i1 = min(T, i0 + step)
        res[:, :, i0:i1] = (w[:, :, i0:i1, :, None] * (v[:, :, None] - o[:, :, i0:i1, None]).abs()).sum(3)
    return res


def attention_ref(qkv: torch.Tensor, B: int, T: int, nh: int, hd: int, scale: float, interleaved: bool = False, nkv: int = -1,
                  out: Optional[torch.Tensor] = None, dout: Optional[torch.Tensor] = None) -> dict:
    """fp64 reference of the extension's ``attention_fwd(qkv, out, lse, B, T, nh, hd, scale, interleaved, nkv)`` and, with
    ``out`` (the bf16 output of the forward, as passed to the backward) and ``dout``, of ``attention_bwd``.  Computed on the
    device of ``qkv``.  Returns ``{name: (ref, bound, score, floor)}`` for ``out``, ``lse`` and, for the backward, ``dq``, ``dk``,
    ``dv``, laid out as :func:`attention_unpack` / :func:`attention_heads` lay out the kernel's buffers (``lse``: ``[B, nh, T]``).

    Query head h of batch b reads KV head κ(h) = h // (nh / nkv) (h itself when interleaved).  For query i and key k ≤ i, all
    from the bf16 inputs as stored:

        s_ik = scale·Σ_d q_id k_kd     σ_ik = |scale|·Σ_d |q_id||k_kd|     P = causal softmax of s     O = P·V
        lse_i = log2 Σ_k exp(s_ik)     (the log2 domain the kernels store)
        dP_ik = Σ_j dO_ij v_kj     Δ_i = Σ_j dO_ij O'_ij     dS_ik = P_ik (dP_ik − Δ_i)
        dQ = scale·dS·K     dK_κ = scale·Σ_{h: κ(h) = κ} dSᵀ·Q     dV_κ = Σ_{h: κ(h) = κ} Pᵀ·dO

    O' is ``out`` as passed: the bf16 rounding of the forward output inside Δ is part of the definition, as it is in the
    kernels, and is not a tolerance term.

    ``bound`` is the magnitude the operand roundings scale with (:func:`assert_attention_close` multiplies it by c_p, c_l or
    c_d):

        out: Σ_k P_ik |v_kj|          P packed to bf16 as the register A operand of O += P·V; ex2.approx; the fp32 row sum
        lse: 1 + |lse_i|              fp32 row maximum and row sum, ex2.approx and log2 of the sum
        dq:  |scale|·Σ_k D_ik |k_kd|  dS packed to bf16 for dQ += dS·K; fp32 dP and Δ (Δ from the bf16 ``out``)
        dk:  |scale|·Σ D_ik |q_id|    dS packed to bf16 for dK += dSᵀ·Q
        dv:  Σ P_ik |dO_ij|           P packed to bf16 for dV += Pᵀ·dO
        with D_ik = P_ik·(Σ_j |dO_ij||v_kj| + Σ_j |dO_ij||O'_ij|) ≥ |dS_ik|, sums over the group's query heads for dk / dv.

    ``score`` is the magnitude the fp32 score error scales with (multiplied by c_s): the scores are accumulated in fp32 and
    rounded again in s·scale·log2(e), an error of up to c_s·σ_ik in s_ik.  It moves O_ij by Σ_k P_ik δs_ik (v_kj − O_ij) and
    lse_i by log2(e)·Σ_k P_ik δs_ik, so

        out: Σ_k P_ik σ_ik |v_kj − O_ij|     lse: log2(e)·Σ_k P_ik σ_ik

    The backward recomputes P from s and the stored lse, so P_ik carries a relative error of up to c_s·ρ_ik with
    ρ_ik = σ_ik + Σ_k' P_ik' σ_ik' (its own score and the lse); the part c_l·(1 + |lse|) of the lse error adds at most
    ln2·c_l·(1 + |lse|) relative, below 2⁻¹⁰ for |lse| < 1000, which c_d covers.  Hence dq: |scale|·Σ_k D_ik ρ_ik |k_kd|,
    dk: |scale|·Σ D_ik ρ_ik |q_id|, dv: Σ P_ik ρ_ik |dO_ij|.

    ``floor`` is the absolute error of flushing fp32 subnormals to zero (ATTN_FTZ = 2⁻¹²⁶ per flushed factor or product): a
    probability, a dS element or a product that underflows loses at most 2⁻¹²⁶ times the other factors of its term, and the
    output itself at most 2⁻¹²⁶.  With A_ik = Σ_j |dO_ij||v_kj| + Σ_j |dO_ij||O'_ij| (≥ |dP_ik − Δ_i|) over the causal k ≤ i:

        out: 2⁻¹²⁶·(1 + Σ_k (1 + |v_kj|))                  lse: 0
        dq:  2⁻¹²⁶·(1 + |scale|·Σ_k (1 + A_ik)(1 + |k_kd|))   dk: 2⁻¹²⁶·(1 + |scale|·Σ (1 + A_ik)(1 + |q_id|))
        dv:  2⁻¹²⁶·(1 + Σ (1 + |dO_ij|))

    It is negligible unless the result itself is below the fp32 normal range (|s| in the hundreds)."""
    nkv = nh if nkv < 0 else nkv
    group = nh // nkv
    q, k, v = attention_unpack(qkv.to(_F64), B, T, nh, hd, nkv=nkv, interleaved=interleaved)
    kvh = torch.arange(nh, device=qkv.device) // group
    kr, vr = k[:, kvh], v[:, kvh]
    causal = torch.ones(T, T, dtype=torch.bool, device=qkv.device).tril()
    s = (scale * (q @ kr.transpose(-1, -2))).masked_fill(~causal, -math.inf)
    sig = (abs(scale) * (q.abs() @ kr.abs().transpose(-1, -2))).masked_fill(~causal, 0.0)
    lse_e = torch.logsumexp(s, -1)
    P = torch.exp(s - lse_e[..., None])
    o = P @ vr
    Psig = P * sig
    cf = causal.to(_F64)
    lse2 = lse_e * _LOG2E
    res = {"out": (o, P @ vr.abs(), _spread(Psig, vr, o), ATTN_FTZ * (1.0 + cf @ (1.0 + vr.abs()))),
           "lse": (lse2, 1.0 + lse2.abs(), _LOG2E * Psig.sum(-1), torch.zeros_like(lse2))}
    if out is None and dout is None:
        return res
    if out is None or dout is None:
        raise ValueError("attention_ref: the backward needs both out and dout")
    Op, dO = attention_heads(out.to(_F64), B, T, nh, hd), attention_heads(dout.to(_F64), B, T, nh, hd)
    dS = P * (dO @ vr.transpose(-1, -2) - (dO * Op).sum(-1, keepdim=True))
    A = dO.abs() @ vr.abs().transpose(-1, -2) + (dO.abs() * Op.abs()).sum(-1, keepdim=True)
    D = P * A
    M = cf * (1.0 + A)
    rho = sig + Psig.sum(-1, keepdim=True)
    Drho, Prho = D * rho, P * rho
    per_kv = lambda x: x.reshape(B, nkv, group, T, hd).sum(2)  # noqa: E731  (query head h = κ·group + g)
    sc = abs(scale)
    tT = lambda x: x.transpose(-1, -2)  # noqa: E731
    res["dq"] = (scale * (dS @ kr), sc * (D @ kr.abs()), sc * (Drho @ kr.abs()), ATTN_FTZ * (1.0 + sc * (M @ (1.0 + kr.abs()))))
    res["dk"] = (per_kv(scale * (tT(dS) @ q)), per_kv(sc * (tT(D) @ q.abs())), per_kv(sc * (tT(Drho) @ q.abs())),
                 ATTN_FTZ * (1.0 + per_kv(sc * (tT(M) @ (1.0 + q.abs())))))
    res["dv"] = (per_kv(tT(P) @ dO), per_kv(tT(P) @ dO.abs()), per_kv(tT(Prho) @ dO.abs()),
                 ATTN_FTZ * (1.0 + per_kv(tT(cf) @ (1.0 + dO.abs()))))
    return res


def assert_attention_close(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, score: torch.Tensor,
                           floor: torch.Tensor) -> float:
    """Element-wise check of one attention result (``name`` in out, lse, dq, dk, dv) against :func:`attention_ref`:

        |got − ref| ≤ c_out·|ref| + c·bound + c_s·score + floor

    ``c_out`` is the output rounding (2⁻⁸ for bf16, 0 for the fp32 lse, whose rounding c_l covers), ``c`` is
    :data:`ATTN_C_P` (out), :data:`ATTN_C_L` (lse) or :data:`ATTN_C_D` (dq, dk, dv), ``c_s`` :data:`ATTN_C_S`.  A NaN fails.
    Returns the worst ratio of error to tolerance (<= 1 when it passes); the failure message names the element
    (b, head, row, col)."""
    g = got.to(_F64)
    c_out = 2.0 ** -8 if got.dtype == torch.bfloat16 else 0.0
    err = (g - ref).abs()
    tol = c_out * ref.abs() + _ATTN_C[name] * bound + ATTN_C_S * score + floor
    ratio = torch.where(tol > 0, err / tol.clamp(min=1e-300), torch.where(err == 0, 0.0, math.inf))
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
    flat = int(torch.argmax(ratio))
    idx = list(torch.unravel_index(torch.tensor(flat), ratio.shape))
    idx = tuple(int(i) for i in idx)
    worst = float(ratio[idx])
    if not worst <= 1.0:
        n_bad = int((ratio > 1.0).sum())
        where = ", ".join(f"{n} {i}" for n, i in zip(("b", "head", "row", "col"), idx))
        raise AssertionError(
            f"attention {name} out of tolerance at {n_bad} of {ratio.numel()} elements; worst ratio {worst:.3g} at ({where}): "
            f"got={float(g[idx]):.6g} ref={float(ref[idx]):.6g} tol={float(tol[idx]):.6g} (bound={float(bound[idx]):.6g}, "
            f"score={float(score[idx]):.6g}, floor={float(floor[idx]):.3g})")
    return worst


# ----------------------------------------------------------------------------- row-wise kernels (csrc/kernels.h)
# fp64 evaluations of the contracts of the norm, rotary, activation, loss, embedding, dropout, fp8 and optimizer kernels, written
# from their documentation.  Each takes the kernel's inputs as stored (and, where a later output is defined in terms of an earlier
# one, the earlier output as the kernel stored it, like O' in attention_ref) and returns, per output, either ``(ref, bound)`` for
# assert_rowwise_close or an exact tensor for assert_bitwise_equal.  ``bound`` already carries its coefficient: it is the
# absolute error allowed beyond the rounding of the output itself.
#
# Intermediate roundings are part of the definitions and are reproduced, not absorbed: the bf16 x̂ of RMSNorm (forward and dw),
# the rounded dz that GELU's dbias sums, the rounded activation that the dropout and E4M3 copies are made from.  Only two
# constants are empirical.  ROW_C_ACC is the fp32 accumulation error of a sum per unit of Σ|terms| (row statistics, dw / db /
# dres_sum / dtable / dbias / sumsq / loss_sum), ROW_C_F32 the error of a few fp32 operations and of rsqrtf, __expf,
# __fdividef, erff, tanhf and powf per unit of the element's magnitude term.  Both are set from the worst element observed
# on an H100 80GB HBM3 (700 W) over tests/test_rowwise_modes_gpu.py (sweep and executor audit; its "calibration" lines with -s
# print each family's share of the coefficient), with headroom: sums reached 2.2e-7·Σ|terms| (share 0.229 of 2^-20, RMSNorm dw at
# M = 1500, H = 8192; LayerNorm dw 0.222) and element-wise fp32 results 9.2e-7 per unit of their magnitude term (share 0.242 of
# 2^-18, LayerNorm rstd at H = 4096 with a mean offset of 64; tanh-GELU dz 0.142).
ROW_C_ACC = 2.0 ** -20
ROW_C_F32 = 2.0 ** -18
# fp32 results below the normal range may be flushed (ex2.approx.ftz inside __expf, __fdividef past 2^126): at most this much
ROW_FTZ = 2.0 ** -126
_BF16_OUT = 2.0 ** -8  # relative rounding of a bf16 output (round to nearest, 8 significant bits)
_F32_OUT = 2.0 ** -24


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float32)


def _bf16_round(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16 -> fp32 with round-to-nearest-even (__float2bfloat16_rn)."""
    return t.to(torch.float32).to(torch.bfloat16).to(torch.float32)


def _seed_of(seed) -> int:
    if seed is None:
        return 0
    return (int(seed.reshape(-1)[0].item()) if torch.is_tensor(seed) else int(seed)) & _M32


def _keep_f32(p: float) -> float:
    """The fp32 ``1/(1-p)`` the bindings pass to the kernels."""
    return float(torch.tensor(1.0 / (1.0 - p), dtype=torch.float32))


def dropout_copy_exact(y: torch.Tensor, seed, key: int, p: float, row_offset: int = 0) -> torch.Tensor:
    """bf16 ``keep ⊙ y · fp32(1/(1-p))`` of a ``[M, H]`` bf16 tensor, mask stream ``mix_seed(seed, key)`` over (row, column),
    product and rounding in fp32 as the kernels do it: the exact expected dropout copy."""
    keep = dropout_keep_mask(mix_seed(_seed_of(seed), key), y.shape[0], y.shape[1], p, device=y.device, row_offset=row_offset)
    return torch.where(keep, _f32(y) * _keep_f32(p), torch.zeros((), device=y.device)).to(torch.bfloat16)


def fp8_saturate(x32: torch.Tensor, e5m2: bool = False) -> torch.Tensor:
    """Saturating round-to-nearest-even of fp32 values to E4M3 (or E5M2), as ``uint8`` bits (``__NV_SATFINITE``)."""
    fmax = 57344.0 if e5m2 else 448.0
    return x32.clamp(-fmax, fmax).to(torch.float8_e5m2 if e5m2 else torch.float8_e4m3fn).view(torch.uint8)


def fp8_copy_exact(y: torch.Tensor, inv_scale: torch.Tensor, amax_before: torch.Tensor, e5m2: bool = False):
    """``(q8, amax)`` of a producer's E4M3 side output from its bf16 primary output ``y``: q8 = sat(fp32(y · inv_scale)),
    amax = max(amax_before, max |y|)."""
    inv = _f32(inv_scale.reshape(-1)[:1]).to(y.device)
    q = fp8_saturate(_f32(y) * inv, e5m2)
    amax = torch.maximum(_f32(amax_before).reshape(-1)[:1].to(y.device), _f32(y).abs().max().reshape(1))
    return q, amax


def rmsnorm_fwd_ref(x: torch.Tensor, w: torch.Tensor, eps: float, rstd_got: torch.Tensor) -> dict:
    """Contract of ``rmsnorm_fwd(x, w, y, rstd, eps, ...)`` on ``x [M, H]``:

        rstd = 1 / sqrt(Σ_j x_j² / H + eps)        (fp32 sum, rsqrtf)          -> ("rstd": ref, bound)
        y    = bf16(w · bf16(fp32(x · rstd)))      with the stored fp32 rstd    -> ("y": exact)

    The inner product x·rstd is one fp32 multiplication and w · bf16(..) is exact in fp32, so given the rstd the kernel stored,
    y has one correct value.  The dropout copies and the E4M3 copy are derived from the stored y (dropout_copy_exact,
    fp8_copy_exact)."""
    X = x.to(_F64)
    r = 1.0 / torch.sqrt((X * X).mean(-1) + eps)
    rs = _f32(rstd_got).reshape(-1, 1)
    xh = _bf16_round(_f32(x) * rs)
    y = (xh * _f32(w).reshape(1, -1)).to(torch.bfloat16)
    return {"rstd": (r, ROW_C_F32 * r), "y": y}


def rmsnorm_bwd_ref(dy, x, w, rstd, dx_add=None, dw_before=None) -> dict:
    """Contract of ``rmsnorm_bwd(dy, x, w, rstd, dx_add, dx, dw)`` with the stored fp32 ``rstd`` (one per row):

        x̂ = x · rstd,   g = dy · w
        dx = rstd · (g − x̂ · Σ_j g_j x̂_j / H) + dx_add                         (fp32, one bf16 rounding)
        dw = dw_before + Σ_rows dy · bf16(fp32(x · rstd))                        (fp32 accumulation)

    The bf16 x̂ inside dw is the one the forward multiplied the weight with; it is reproduced exactly."""
    rs = _f32(rstd).reshape(-1, 1)
    X, DY, W, RS = x.to(_F64), dy.to(_F64), w.to(_F64).reshape(1, -1), rs.to(_F64)
    H = X.shape[1]
    xh = X * RS
    g = DY * W
    dot = (g * xh).sum(-1, keepdim=True) / H
    adot = (g * xh).abs().sum(-1, keepdim=True) / H
    dx = RS * (g - xh * dot)
    bdx = RS * (g.abs() + xh.abs() * adot)
    if dx_add is not None:
        dx = dx + dx_add.to(_F64)
        bdx = bdx + dx_add.to(_F64).abs()
    xhb = _bf16_round(_f32(x) * rs).to(_F64)
    t = DY * xhb
    dw0 = torch.zeros(H, dtype=_F64, device=x.device) if dw_before is None else dw_before.to(_F64)
    return {"dx": (dx, ROW_C_F32 * bdx), "dw": (dw0 + t.sum(0), ROW_C_ACC * (dw0.abs() + t.abs().sum(0)))}


def layernorm_fwd_ref(x, eps: float, mean_got, rstd_got, norms) -> dict:
    """Contract of ``layernorm_fwd(x, w, b, y, mean, rstd, eps, w2, b2, y2, ...)`` on ``x [M, H]``:

        mean = Σ x / H                                  (fp32)                   -> ("mean": ref, bound)
        rstd = 1 / sqrt(Σ (x − mean)² / H + eps)        two-pass, the stored mean -> ("rstd": ref, bound)
        y_n  = (x − mean) · rstd · w_n + b_n            stored mean / rstd, fp32, one bf16 rounding -> ("y0", "y1")

    ``norms``: list of ``(w, b or None)``.  The dropout copies are derived from the stored y (dropout_copy_exact)."""
    X = x.to(_F64)
    H = X.shape[1]
    mu = X.mean(-1)
    m_got = _f32(mean_got).to(_F64).reshape(-1, 1)
    var = ((X - m_got) ** 2).mean(-1)
    r = 1.0 / torch.sqrt(var + eps)
    res = {"mean": (mu, ROW_C_F32 * X.abs().mean(-1)), "rstd": (r, ROW_C_F32 * r)}
    rs = _f32(rstd_got).to(_F64).reshape(-1, 1)
    for n, (w, b) in enumerate(norms):
        W = w.to(_F64).reshape(1, -1)
        B = b.to(_F64).reshape(1, -1) if b is not None else torch.zeros(1, H, dtype=_F64, device=x.device)
        xh = (X - m_got) * rs
        res[f"y{n}"] = (xh * W + B, ROW_C_F32 * ((xh * W).abs() + B.abs()))
    return res


def layernorm_bwd_ref(x, mean, rstd, norms, dres=None, dres_sums=()) -> dict:
    """Contract of ``layernorm_bwd`` with the stored fp32 ``mean`` / ``rstd``; ``norms``: list of ``(dy, w, dw_before,
    db_before or None)`` (one, or two for the dual form):

        x̂ = (x − mean) · rstd,   g_n = dy_n · w_n
        dx  = dres + Σ_n rstd · (g_n − Σ_j g_n,j / H − x̂ · Σ_j g_n,j x̂_j / H)      (fp32, one bf16 rounding)
        dw_n = dw_before + Σ_rows dy_n · x̂      db_n = db_before + Σ_rows dy_n
        dres_sum_k = before_k + Σ_rows dres  for each ``before_k`` in ``dres_sums``"""
    X = x.to(_F64)
    H = X.shape[1]
    xh = (X - _f32(mean).to(_F64).reshape(-1, 1)) * _f32(rstd).to(_F64).reshape(-1, 1)
    RS = _f32(rstd).to(_F64).reshape(-1, 1)
    dx = torch.zeros_like(X) if dres is None else dres.to(_F64)
    bdx = torch.zeros_like(X) if dres is None else dres.to(_F64).abs()
    res = {}
    for n, (dy, w, dw0, db0) in enumerate(norms):
        DY = dy.to(_F64)
        g = DY * w.to(_F64).reshape(1, -1)
        sg, sgx = g.sum(-1, keepdim=True) / H, (g * xh).sum(-1, keepdim=True) / H
        dx = dx + RS * (g - sg - xh * sgx)
        bdx = bdx + RS * (g.abs() + g.abs().sum(-1, keepdim=True) / H + xh.abs() * (g * xh).abs().sum(-1, keepdim=True) / H)
        for name, before, t in ((f"dw{n}", dw0, DY * xh), (f"db{n}", db0, DY)):
            if before is not None:
                b0 = before.to(_F64)
                res[name] = (b0 + t.sum(0), ROW_C_ACC * (b0.abs() + t.abs().sum(0)))
    res["dx"] = (dx, ROW_C_F32 * bdx)
    for k, before in enumerate(dres_sums):
        b0, D = before.to(_F64), dres.to(_F64)
        res[f"dres_sum{k}"] = (b0 + D.sum(0), ROW_C_ACC * (b0.abs() + D.abs().sum(0)))
    return res


def cross_entropy_ref(logits: torch.Tensor, labels: torch.Tensor, V: int, grad_scale: float, ignore_index: int,
                      loss_before, count_before) -> dict:
    """Contract of ``cross_entropy_fwd_bwd(logits, labels, V, grad_scale, ignore_index, loss_sum, count)`` on the bf16
    ``logits[:, :V]`` as stored (row pitch ≥ V; the columns [V, ld) are neither read nor written):

        row with label y ≠ ignore_index:  lse = log Σ_j exp(x_j),  loss_sum += lse − x_y,  count += 1
                                          x_j <- bf16(grad_scale · (softmax_j − [j = y]))
        ignored row:                      x_j <- 0 exactly

    Bounds with m the row maximum and ρ_j = 1 + |x_j − m| (__expf's argument is rounded relative to its size): the gradient
    ROW_C_F32·|gs|·p_j·(ρ_j + Σ_k p_k ρ_k) + |gs|·ROW_FTZ, the loss ROW_C_F32·(|lse| + |m| + |x_y| + Σ_k p_k ρ_k) per row plus
    ROW_C_ACC over the rows' sum.  ``count`` is exact."""
    X = logits[:, :V].to(_F64)
    lab = labels.to(torch.int64).reshape(-1).to(X.device)
    valid = lab != ignore_index
    m = X.max(-1, keepdim=True).values
    e = torch.exp(X - m)
    se = e.sum(-1, keepdim=True)
    P = e / se
    lse = m + torch.log(se)
    rho = 1.0 + (X - m).abs()
    prho = (P * rho).sum(-1, keepdim=True)
    onehot = torch.zeros_like(X)
    lab_c = lab.clamp(0, V - 1)
    onehot.scatter_(1, lab_c.view(-1, 1), 1.0)
    gs = float(grad_scale)
    vm = valid.view(-1, 1).to(_F64)
    grad = gs * (P - onehot) * vm
    bgrad = (ROW_C_F32 * abs(gs) * P * (rho + prho) + abs(gs) * ROW_FTZ) * vm
    xl = X.gather(1, lab_c.view(-1, 1))
    row_loss = ((lse - xl) * vm).reshape(-1)
    row_b = (ROW_C_F32 * (lse.abs() + m.abs() + xl.abs() + prho) * vm).reshape(-1)
    l0 = _f32(loss_before).reshape(-1)[0].to(_F64)
    total = l0 + row_loss.sum()
    loss_bound = ROW_C_ACC * (l0.abs() + (row_loss.abs()).sum()) + row_b.sum()
    count = _f32(count_before).reshape(-1)[0] + float(int(valid.sum()))
    return {"grad": (grad, bgrad), "loss_sum": (total.reshape(1), loss_bound.reshape(1)), "count": count.reshape(1)}


def _rotate(a, b, c, s):
    """(a c − b s, b c + a s) and its magnitude (|a c| + |b s|, |b c| + |a s|) in fp64."""
    return a * c - b * s, b * c + a * s, (a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()


def rope_inplace_ref(buf: torch.Tensor, T: int, n_rot_heads: int, hd: int, rotary_dim: int, cos, sin, backward: bool, pos0: int):
    """Contract of ``rope_inplace(buf, T, n_rot_heads, hd, rotary_dim, cos, sin, backward, pos0)`` on ``buf [M, ≥ n_rot_heads·hd]``
    as it was before the call.  Row r sits at position r mod T + pos0; head h < n_rot_heads, i < rotary_dim/2:

        (a, b) = (x[h·hd + i], x[h·hd + i + rotary_dim/2]) -> (a c − b s, b c + a s),  c = cos[pos, i],  s = ±sin[pos, i]

    (s negated for the backward), in fp32 with one bf16 rounding.  Returns ``(mask, ref, bound)`` over buf's columns: where
    ``mask`` is False the element must keep its bits."""
    return _rope_ref(buf, T, [h * hd for h in range(n_rot_heads)], rotary_dim, cos, sin, -1.0 if backward else 1.0, pos0)


def _rope_ref(buf, T, starts, rot, cos, sin, sgn, pos0):
    X = buf.to(_F64)
    M, W = X.shape
    half = rot // 2
    pos = torch.arange(M, device=buf.device) % T + pos0
    c = cos.to(_F64)[pos][:, :half]
    s = sgn * sin.to(_F64)[pos][:, :half]
    ref, bound = X.clone(), torch.zeros_like(X)
    mask = torch.zeros(M, W, dtype=torch.bool, device=buf.device)
    for s0 in starts:
        a, b = X[:, s0:s0 + half], X[:, s0 + half:s0 + rot]
        y1, y2, b1, b2 = _rotate(a, b, c, s)
        ref[:, s0:s0 + half], ref[:, s0 + half:s0 + rot] = y1, y2
        bound[:, s0:s0 + half], bound[:, s0 + half:s0 + rot] = ROW_C_F32 * b1, ROW_C_F32 * b2
        mask[:, s0:s0 + rot] = True
    return mask, ref, bound


def neox_rope_ref(qkv: torch.Tensor, T: int, nh: int, hd: int, rot: int, cos, sin, pos0: int, inverse: bool):
    """Contract of ``neox_rope(qkv, T, nh, hd, rot, cos, sin, pos0, inverse)`` on the GPT-NeoX ``[rows, nh·(q|k|v)·hd]`` layout
    with fp32 tables ``[n_pos, rot]``: the first ``rot`` dims of each q and k head rotate as in :func:`rope_inplace_ref`; v and
    the dims past ``rot`` keep their bits.  Returns ``(mask, ref, bound)``."""
    starts = [h * 3 * hd + w * hd for h in range(nh) for w in (0, 1)]
    return _rope_ref(qkv, T, starts, rot, cos, sin, -1.0 if inverse else 1.0, pos0)


def rope_pack_bwd_ref(dq, dk, dv, rotary_dim: int, cos, sin, pos0: int):
    """Contract of ``rope_pack_bwd(dq, dk, dv, out, rotary_dim, cos, sin, pos0, nkv)``: ``dq [B, nh, T, hd]``, ``dk / dv
    [B, nkv, T, hd]`` (any strides) gathered into ``out [B·T, (nh + 2·nkv)·hd]`` = [q heads | k heads | v heads], q and k
    rotated back (s -> −s, position t + pos0) in their first ``rotary_dim`` dims, everything else copied.  Returns
    ``(exact_mask, ref, bound)``: where ``exact_mask`` is set the value is a copy and must match bit for bit."""
    B, nh, T, hd = dq.shape
    nkv = dk.shape[1]
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(B * T, -1)  # noqa: E731  [B·T, heads·hd]
    X = torch.cat([rows(dq), rows(dk), rows(dv)], 1)
    mask, ref, bound = _rope_ref(X, T, [h * hd for h in range(nh + nkv)], rotary_dim, cos, sin, -1.0, pos0)
    return ~mask, ref, bound


def swiglu_fwd_ref(gu: torch.Tensor, F: int) -> tuple:
    """Contract of ``swiglu_fwd(gu, h, ...)``: ``h = bf16(silu(g) · u)`` with g = gu[:, :F], u = gu[:, F:2F], computed as
    g / (1 + __expf(−g)) · u.  Bound ROW_C_F32·|h|·(1 + |g|) (__expf's argument); where 1 + e^{−g} passes 2^126 (g < −87)
    __fdividef returns 0, so there the whole value is allowed.  The dropout / E4M3 copies are derived from the stored h."""
    G, U = gu[:, :F].to(_F64), gu[:, F:2 * F].to(_F64)
    sg = torch.sigmoid(G)
    h = G * sg * U
    bound = ROW_C_F32 * h.abs() * (1.0 + G.abs()) + torch.where(G < -87.0, h.abs(), torch.zeros_like(h))
    return h, bound


def swiglu_bwd_ref(dh: torch.Tensor, gu: torch.Tensor, F: int) -> dict:
    """Contract of ``swiglu_bwd(dh, gu, dgu)``: with σ = sigmoid(g), silu = g·σ (σ = __fdividef(1, 1 + __expf(−g))):

        dgu[:, :F] = dh · u · (σ + silu · (1 − σ))        dgu[:, F:] = dh · silu

    Bounds as :func:`swiglu_fwd_ref` (magnitudes σ(1 + |g|(1 − σ))·|dh u| and |dh silu|)."""
    G, U, D = gu[:, :F].to(_F64), gu[:, F:2 * F].to(_F64), dh.to(_F64)
    sg = torch.sigmoid(G)
    silu = G * sg
    dg = D * U * (sg + silu * (1.0 - sg))
    du = D * silu
    flush = G < -87.0
    z = torch.zeros_like(dg)
    bdg = ROW_C_F32 * (D * U).abs() * sg * (1.0 + G.abs() * (1.0 - sg)) * (1.0 + G.abs()) + torch.where(flush, dg.abs(), z)
    bdu = ROW_C_F32 * du.abs() * (1.0 + G.abs()) + torch.where(flush, du.abs(), z)
    return {"dg": (dg, bdg), "du": (du, bdu)}


_SQRT_2_OVER_PI = math.sqrt(2.0 / math.pi)


def gelu_fwd_ref(z: torch.Tensor, tanh_approx: bool) -> tuple:
    """Contract of ``gelu_fwd(z, a, tanh_approx)``: a = bf16(0.5 z (1 + erf(z/√2))), or with the tanh form
    0.5 z (1 + tanh(√(2/π)(z + 0.044715 z³))), fp32 erff / tanhf.  The absolute error of 1 + erf (or 1 + tanh) is a few fp32
    ulps of 1 (and, for tanh, of the argument u times 1 − t²), so the bound is ROW_C_F32·0.5|z|·(1 + |u|(1 − t²))."""
    Z = z.to(_F64)
    if tanh_approx:
        u = _SQRT_2_OVER_PI * (Z + 0.044715 * Z ** 3)
        t = torch.tanh(u)
        a = 0.5 * Z * (1.0 + t)
        mag = 0.5 * Z.abs() * (1.0 + u.abs() * (1.0 - t * t))
    else:
        a = 0.5 * Z * torch.erfc(-Z / math.sqrt(2.0))  # 1 + erf without its cancellation for z << 0
        mag = 0.5 * Z.abs() * 2.0
    return a, ROW_C_F32 * (mag + a.abs())


def gelu_bwd_ref(da: torch.Tensor, z: torch.Tensor, tanh_approx: bool) -> tuple:
    """Contract of ``gelu_bwd(da, z, dz, tanh_approx)``: dz = bf16(da · GELU'(z)); erf form
    GELU'(z) = 0.5 (1 + erf(z/√2)) + z φ(z) with φ from __expf(−z²/2), tanh form
    0.5 (1 + t) + 0.5 z (1 − t²) √(2/π)(1 + 3·0.044715 z²).  Bound ROW_C_F32·|da|·(1 + |z|·d(z)·(1 + z²)), d the size of the
    exponential / sech² factor.  ``dbias`` (column sum of the *rounded* dz) is checked with :func:`colsum_ref` on the dz the
    kernel stored."""
    Z, DA = z.to(_F64), da.to(_F64)
    if tanh_approx:
        u = _SQRT_2_OVER_PI * (Z + 0.044715 * Z ** 3)
        t = torch.tanh(u)
        d = 0.5 * (1.0 + t) + 0.5 * Z * (1.0 - t * t) * _SQRT_2_OVER_PI * (1.0 + 3.0 * 0.044715 * Z * Z)
        fac = (1.0 - t * t) * (1.0 + u.abs())
    else:
        phi = torch.exp(-0.5 * Z * Z) / math.sqrt(2.0 * math.pi)
        d = 0.5 * torch.erfc(-Z / math.sqrt(2.0)) + Z * phi
        fac = phi
    return DA * d, ROW_C_F32 * DA.abs() * (1.0 + Z.abs() * fac * (1.0 + Z * Z))


def colsum_ref(x: torch.Tensor, before: torch.Tensor) -> tuple:
    """``out = before + Σ_rows x`` (``colsum``, the dbias of ``gelu_bwd`` over the stored dz), fp32 accumulation."""
    X, b0 = x.to(_F64), before.to(_F64)
    return b0 + X.sum(0), ROW_C_ACC * (b0.abs() + X.abs().sum(0))


def embedding_bwd_ref(ids: torch.Tensor, dout: torch.Tensor, dtable_before: torch.Tensor, padding_idx: int) -> tuple:
    """``embedding_bwd``: dtable[id] += dout row for every position whose id is not ``padding_idx`` (fp32 atomics)."""
    idx = ids.reshape(-1).to(torch.int64)
    D = dout.reshape(idx.numel(), -1).to(_F64)
    keep = idx != padding_idx
    acc = torch.zeros(dtable_before.shape, dtype=_F64, device=D.device)
    mag = torch.zeros_like(acc)
    acc.index_add_(0, idx[keep], D[keep])
    mag.index_add_(0, idx[keep], D[keep].abs())
    b0 = dtable_before.to(_F64)
    return b0 + acc, ROW_C_ACC * (b0.abs() + mag)


def embedding_bwd_sorted_exact(sorted_ids: torch.Tensor, perm: torch.Tensor, dout: torch.Tensor, dtable_before: torch.Tensor,
                               padding_idx: int) -> torch.Tensor:
    """``embedding_bwd_sorted(sorted_ids, perm, dout, dtable, padding_idx)``: for every run of equal ids in ``sorted_ids``, the
    fp32 sum of the rows ``dout[perm[k]]`` in run order starting from 0, then one fp32 add into the prior table row (a stable
    sort makes the run order the position order).  Plain fp32 adds, no FMA: reproduced bit for bit."""
    sid = sorted_ids.reshape(-1).to(torch.int64).cpu()
    pm = perm.reshape(-1).to(torch.int64).cpu()
    D = _f32(dout.reshape(sid.numel(), -1)).cpu()
    out = _f32(dtable_before).cpu().clone()
    uniq, counts = torch.unique_consecutive(sid, return_counts=True)
    starts = torch.cumsum(counts, 0) - counts
    sel = uniq != padding_idx
    uniq, counts, starts = uniq[sel], counts[sel], starts[sel]
    acc = torch.zeros(uniq.numel(), D.shape[1], dtype=torch.float32)
    for k in range(int(counts.max()) if counts.numel() else 0):
        live = counts > k
        acc[live] = acc[live] + D[pm[starts[live] + k]]
    out[uniq] = out[uniq] + acc
    return out.to(dtable_before.device)


def dropout_combine_ref(base, parts_groups, seed, keys, p: float) -> tuple:
    """``dropout_combine(base, parts, out, seed, keys, p)``: out = bf16(base + Σ_g keep_g ⊙ parts_g / (1 − p)), fp32."""
    M, H = parts_groups[0].shape
    acc = torch.zeros(M, H, dtype=_F64, device=parts_groups[0].device) if base is None else base.to(_F64).reshape(M, H)
    mag = acc.abs()
    inv = _keep_f32(p)
    for g, part in enumerate(parts_groups):
        keep = dropout_keep_mask(mix_seed(_seed_of(seed), keys[g]), M, H, p, device=part.device)
        t = part.to(_F64) * inv * keep
        acc, mag = acc + t, mag + t.abs()
    return acc, ROW_C_F32 * mag


def adamw_ref(p, g, m, v, *, lr, b1, b2, eps, wd, step, grad_scale: float = 1.0) -> dict:
    """Contract of ``adamw_flat(p, g, m, v, lr, b1, b2, eps, wd, step, grad_scale, grad_scale_host, skip, step_dev)`` with the
    hyperparameters as the fp32 values the kernel receives and ``grad_scale`` the product of the device and host scales:

        g' = g·gs,  m' = b1 m + (1 − b1) g',  v' = b2 v + (1 − b2) g'²              (stored in m's / v's dtype)
        p' = bf16(p (1 − lr wd) − lr/(1 − b1^t) · m' / (√v' / √(1 − b2^t) + eps))    (from the unrounded m', v')

    Bounds: ROW_C_F32 times the magnitudes of the terms; powf's relative error ε (inside ROW_C_F32) in b^t becomes
    ε·b^t/(1 − b^t) in the bias corrections, which is large at small t, so that factor is carried explicitly."""
    f = lambda a: float(torch.tensor(a, dtype=torch.float32))  # noqa: E731
    lr, b1, b2, eps, wd, gs = f(lr), f(b1), f(b2), f(eps), f(wd), f(grad_scale)
    G, P, Mo, Vo = g.to(_F64) * gs, p.to(_F64), m.to(_F64), v.to(_F64)
    m1 = b1 * Mo + (1.0 - b1) * G
    v1 = b2 * Vo + (1.0 - b2) * G * G
    bm = b1 * Mo.abs() + (1.0 - b1) * G.abs()
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    k1, k2 = 1.0 + b1 ** step / bc1, 1.0 + b2 ** step / bc2
    denom = torch.sqrt(v1) / math.sqrt(bc2) + eps
    upd = (lr / bc1) * m1 / denom
    decay = 1.0 - lr * wd
    pn = P * decay - upd
    bp = ROW_C_F32 * (P.abs() * abs(decay) + (lr / bc1) * bm / denom * (k1 + k2))
    return {"p": (pn, bp), "m": (m1, ROW_C_F32 * bm), "v": (v1, ROW_C_F32 * v1)}


def sumsq_ref(x: torch.Tensor, before: torch.Tensor) -> tuple:
    """``sumsq(x, out)``: out = before + Σ x², fp32 accumulation."""
    X, b0 = x.to(_F64).reshape(-1), _f32(before).reshape(-1)[:1].to(_F64)
    s = (X * X).sum()
    return b0 + s, ROW_C_ACC * (b0.abs() + s)


def fp8_quantize_weight_exact(w: torch.Tensor):
    """``fp8_quantize_weight(w, w8, scratch, scale, inv_scale, w8t)``: amax = max|w|, scale = max(amax, 1e-12)/448,
    inv_scale = 1/scale (IEEE fp32), w8 = sat_e4m3(fp32(w · inv_scale)), w8t its transpose.  Returns the exact
    ``(amax, scale, inv_scale, w8, w8t)``."""
    W = _f32(w)
    amax = W.abs().max().reshape(1)
    # numpy: a torch division by a Python scalar multiplies by the reciprocal, one ulp off the kernel's IEEE division
    a = amax.cpu().numpy()
    scale = np.maximum(a, np.float32(1e-12)) / np.float32(448.0)
    inv = np.float32(1.0) / scale
    scale, inv = torch.from_numpy(scale).to(w.device), torch.from_numpy(inv).to(w.device)
    q = fp8_saturate(W * inv)
    return amax, scale, inv, q, q.t().contiguous()


def fp8_prep_exact(state, w_scale, margin: float, n_e4m3: int) -> dict:
    """``fp8_prep(state, w_scale, inv_sx, alpha_main, alpha_inv, margin, n_e4m3)`` per site i (all fp32, IEEE division):

        prev = state[i,1] > 0 ? state[i,1] : state[i,0];   state[i] <- (prev, 0)
        sx = max(prev, 1e-12) · margin / fmax_i   (fmax 448 for i < n_e4m3, else 57344)
        inv_sx = 1/sx,  alpha_main = sx · w_scale[i],  alpha_inv = 1/alpha_main"""
    S = _f32(state).reshape(-1, 2)
    n = S.shape[0]
    cur, old = S[:, 1], S[:, 0]
    prev = torch.where(cur > 0, cur, old)
    fmax = torch.where(torch.arange(n, device=S.device) < n_e4m3, torch.tensor(448.0, device=S.device),
                       torch.tensor(57344.0, device=S.device))
    sx = torch.clamp(prev, min=torch.tensor(1e-12, dtype=torch.float32, device=S.device)) * torch.tensor(
        margin, dtype=torch.float32) / fmax
    one = torch.tensor(1.0, dtype=torch.float32, device=S.device)
    a = sx * _f32(w_scale).reshape(-1)
    return {"state": torch.stack([prev, torch.zeros_like(prev)], 1).reshape(state.shape), "inv_sx": one / sx,
            "alpha_main": a, "alpha_inv": one / a}


def assert_rowwise_close(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """Element-wise check of a row-wise kernel output against its fp64 contract:

        |got − ref| ≤ c_out·|ref| + bound

    ``c_out`` is the output rounding (2⁻⁸ for bf16, 2⁻²⁴ for fp32); ``bound`` comes from the ``*_ref`` function with its
    coefficient applied.  A NaN fails.  Returns the worst ratio of error to tolerance (<= 1 when it passes); the failure
    message names the worst element by index."""
    g = got.to(_F64)
    ref = ref.to(g.device).expand_as(g)
    bound = bound.to(g.device).expand_as(g)
    c_out = _BF16_OUT if got.dtype == torch.bfloat16 else _F32_OUT
    err = (g - ref).abs()
    tol = c_out * ref.abs() + bound
    ratio = torch.where(tol > 0, err / tol.clamp(min=1e-300), torch.where(err == 0, 0.0, math.inf))
    ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
    if ratio.numel() == 0:
        return 0.0
    flat = int(torch.argmax(ratio))
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), ratio.shape))
    worst = float(ratio[idx])
    if not worst <= 1.0:
        n_bad = int((ratio > 1.0).sum())
        raise AssertionError(
            f"{name} out of tolerance at {n_bad} of {ratio.numel()} elements; worst ratio {worst:.3g} at {idx}: "
            f"got={float(g[idx]):.6g} ref={float(ref[idx]):.6g} tol={float(tol[idx]):.6g} (bound={float(bound[idx]):.6g})")
    return worst


def rowwise_excess(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """Worst (|got − ref| − c_out·|ref|)⁺ / bound: how much of the empirical coefficient inside ``bound`` an output used."""
    g = got.to(_F64)
    c_out = _BF16_OUT if got.dtype == torch.bfloat16 else _F32_OUT
    ex = ((g - ref.to(g.device)).abs() - c_out * ref.to(g.device).abs()).clamp(min=0)
    b = bound.to(g.device).expand_as(ex)
    r = torch.where(b > 0, ex / b.clamp(min=1e-300), torch.zeros_like(ex))
    return float(r.max()) if r.numel() else 0.0


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def assert_bitwise_equal(name: str, got: torch.Tensor, ref: torch.Tensor) -> None:
    """Exact contracts: every element of ``got`` has the bits of ``ref``; the message names the first one that does not."""
    ref = ref.to(got.device)
    if got.shape != ref.shape or got.dtype != ref.dtype:
        raise AssertionError(f"{name}: got {tuple(got.shape)} {got.dtype}, expected {tuple(ref.shape)} {ref.dtype}")
    diff = _bits(got) != _bits(ref)
    if bool(diff.any()):
        idx = tuple(int(i) for i in diff.nonzero()[0])
        n_bad = int(diff.sum())
        gv = got[idx].float().item() if got.is_floating_point() else got[idx].item()
        rv = ref[idx].float().item() if ref.is_floating_point() else ref[idx].item()
        raise AssertionError(f"{name} differs at {n_bad} of {got.numel()} elements; first at {idx}: got={gv!r} expected={rv!r}")


# ----------------------------------------------------------------------------- block-scaled MXFP8 (csrc/gemm_mx.cu)
# Exact contracts of mx_quantize_rows, mx_quantize_weight_2d, mx_dequantize_weight and gemm_mx.  E4M3 elements, one UE8M0 scale
# byte b (value 2^(b-127)) per 32 elements of the reduction dimension: per (row, 32 columns) for activations, per 32 x 32 tile for
# weights (written once in the forward layout, rows N, and once in the backward layout, rows K).
#
#   exponent  e = the smallest integer with amax <= 448·2^e, clamped to [-127, 127]; amax = max |x| over the block, NaN elements
#             ignored (an all-zero or all-NaN block gets -127)
#   elements  RNE(x·2^-e) to E4M3, saturated to ±448; a NaN element gives an E4M3 NaN byte (sign unspecified)
#   ±Inf      a block holding an infinity gets the OCP MX NaN scale 0xFF, decoded as Inf, so every product it feeds is
#             non-finite; its elements are x·0 (zeros, NaN for the infinities).  Other blocks are unaffected.
MX_SF_NAN = 0xFF


def mx_sf_bytes(rows: int, k: int) -> int:
    """Bytes of the scale array of a ``[rows, k]`` operand: 512 per block of 128 rows x 128 reduction elements."""
    return (rows + 127) // 128 * ((k + 127) // 128) * 512


def mx_sf_offset(row, sfcol, kg):
    """Byte offset of the scale of (``row``, scale column ``sfcol``) with ``kg`` groups of 4 scale columns per 128-row block:
    blocks ordered [row block][k group], inside a block byte (r % 32)·16 + (r // 32)·4 + j with r = row % 128, j = sfcol % 4.
    Integers or integer tensors."""
    r = row % 128
    return ((row // 128) * kg + sfcol // 4) * 512 + (r % 32) * 16 + (r // 32) * 4 + sfcol % 4


def _pad128(n: int) -> int:
    return (n + 127) // 128 * 128


def _sf_index(rows: int, k: int, device=None) -> torch.Tensor:
    """``[pad128(rows), pad128(k)/32]`` byte offsets of every scale of a ``[rows, k]`` operand (the array is exactly covered)."""
    r = torch.arange(_pad128(rows), device=device).unsqueeze(1)
    j = torch.arange(_pad128(k) // 32, device=device).unsqueeze(0)
    return mx_sf_offset(r, j, _pad128(k) // 128)


def mx_scale_grid(sf: torch.Tensor, rows: int, k: int) -> torch.Tensor:
    """The scale bytes of a ``[rows, k]`` operand as a ``[pad128(rows), pad128(k)/32]`` grid."""
    return sf.reshape(-1)[_sf_index(rows, k, sf.device)]


def mx_scale_pack(grid: torch.Tensor, rows: int, k: int) -> torch.Tensor:
    """Inverse of :func:`mx_scale_grid`: the ``mx_sf_bytes(rows, k)`` array holding ``grid``."""
    sf = torch.empty(mx_sf_bytes(rows, k), dtype=torch.uint8, device=grid.device)
    sf[_sf_index(rows, k, grid.device)] = grid.to(torch.uint8)
    return sf


def mx_scale_exponent(amax: torch.Tensor) -> torch.Tensor:
    """int64 e: the smallest integer with ``amax <= 448·2^e``, clamped to [-127, 127], for finite ``amax >= 0``.  Exact: with
    amax = m·2^x (m in [0.5, 1), frexp), 448·2^(x-9) = 0.875·2^x and 448·2^(x-8) = 1.75·2^x bracket it, and the comparison with
    448·2^e is exact in fp64."""
    a = amax.to(_F64)
    _, x = torch.frexp(a)
    e0 = x.to(torch.int64) - 9
    e = e0 + (a > torch.ldexp(torch.full_like(a, 448.0), e0)).to(torch.int64)
    return torch.where(a > 0, e, torch.full_like(e, -127)).clamp(-127, 127)


def mx_encode_blocks(v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Blocks ``v [..., 32]`` (values as the kernel holds them in fp32) -> (E4M3 bytes ``[..., 32]``, scale bytes ``[...]``)."""
    v = v.to(_F64)
    amax = torch.where(torch.isnan(v), torch.zeros_like(v), v.abs()).amax(-1)
    inf = torch.isinf(amax)
    e = mx_scale_exponent(torch.where(inf, torch.zeros_like(amax), amax))
    inv = torch.where(inf, torch.zeros_like(amax), torch.ldexp(torch.ones_like(amax), -e))
    # x·2^-e is exact in fp64; where it is not exact in fp32 (below 2^-126) it rounds to ±0 in E4M3 either way
    q = fp8_saturate((v * inv.unsqueeze(-1)).to(torch.float32))
    return q, torch.where(inf, torch.full_like(e, MX_SF_NAN), e + 127).to(torch.uint8)


def mx_quantize_rows_exact(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``mx_quantize_rows(x, q, sf)`` of a bf16 ``[M, K]``: ``(q [M, Kpad], sf)`` byte for byte, Kpad = K rounded up to 128.
    Columns past K are quantised as zeros (padding bytes 0) and rows up to the next multiple of 128 get scales (of zero rows)."""
    M, K = x.shape
    Mp, Kp = _pad128(M), _pad128(K)
    v = torch.zeros(Mp, Kp, dtype=_F64, device=x.device)
    v[:M, :K] = x.to(_F64)
    q, s = mx_encode_blocks(v.view(Mp, Kp // 32, 32))
    return q.view(Mp, Kp)[:M].contiguous(), mx_scale_pack(s, M, K)


def mx_decode(q: torch.Tensor, sf: torch.Tensor, rows: int, k: int) -> torch.Tensor:
    """Exact fp64 values ``[rows, pad128(k)]`` of a K-major packed operand: E4M3(q[r, c]) · 2^(scale(r, c/32) - 127), scale byte
    0xFF read as Inf."""
    Kp = _pad128(k)
    g = mx_scale_grid(sf, rows, k)[:rows].to(_F64)
    s = torch.where(g == MX_SF_NAN, torch.full_like(g, math.inf), torch.exp2(g - 127.0))
    e = q[:rows, :Kp].contiguous().view(torch.float8_e4m3fn).to(_F64)
    return (e.view(rows, Kp // 32, 32) * s.unsqueeze(-1)).view(rows, Kp)


def mx_decode_rows(q: torch.Tensor, sf: torch.Tensor, M: int, K: int) -> torch.Tensor:
    """Exact fp64 ``[M, K]`` values of the output of ``mx_quantize_rows``."""
    return mx_decode(q, sf, M, K)[:, :K]


def mx_decode_weight(q: torch.Tensor, sf_fwd: torch.Tensor, N: int, K: int) -> torch.Tensor:
    """Exact fp64 ``[N, K]`` values of a packed weight (the contract of ``mx_dequantize_weight`` before its bf16 rounding)."""
    return mx_decode(q, sf_fwd, N, K)[:, :K]


def mx_quantize_weight_2d_exact(w: Optional[torch.Tensor] = None, q_old: Optional[torch.Tensor] = None,
                                sf_old: Optional[torch.Tensor] = None, delta: Optional[torch.Tensor] = None, *,
                                N: Optional[int] = None, K: Optional[int] = None):
    """``mx_quantize_weight_2d(w, delta, q, sf_fwd, sf_bwd, N, K)``: ``(q [Npad, Kpad], sf_fwd, sf_bwd)`` byte for byte.

    The source is the bf16 ``w [N, K]``, or (``w`` None, the merge) the packed ``q_old [>= N, >= Kpad]`` / ``sf_old`` (forward
    layout) decoded in fp32 over all Kpad columns; the fp32 ``delta [N, K]`` is then added in fp32.  Rows past N are zeros.
    Each 32 x 32 tile is one block; its scale goes to (row n, column k/32) of ``sf_fwd`` and (row k, column n/32) of ``sf_bwd``."""
    src = w if w is not None else delta
    N = src.shape[0] if N is None else N
    K = src.shape[1] if K is None else K
    Np, Kp = _pad128(N), _pad128(K)
    dev = (w if w is not None else q_old).device
    v = torch.zeros(Np, Kp, dtype=torch.float32, device=dev)
    if w is not None:
        v[:N, :K] = w.to(torch.float32)
    else:
        v[:N] = mx_decode(q_old, sf_old, N, K).to(torch.float32)  # E4M3 value · power of two: exact in fp32
    if delta is not None:
        v[:N, :K] += delta.to(torch.float32)
    tiles = v.view(Np // 32, 32, Kp // 32, 32).permute(0, 2, 1, 3)  # [tn, tk, n, k]
    q, s = mx_encode_blocks(tiles.reshape(Np // 32, Kp // 32, 1024))
    q = q.view(Np // 32, Kp // 32, 32, 32).permute(0, 2, 1, 3).reshape(Np, Kp)
    s_fwd = s.repeat_interleave(32, 0)  # [Np, Kp/32]: row n, column tk
    s_bwd = s.t().repeat_interleave(32, 0)  # [Kp, Np/32]: row k, column tn
    return q, mx_scale_pack(s_fwd, N, K), mx_scale_pack(s_bwd, K, N)


def gemm_mx_ref(a: torch.Tensor, sfa: torch.Tensor, b: torch.Tensor, sfb: torch.Tensor, M: int, N: int, K: int,
                b_mn_major: bool = False, a2: Optional[torch.Tensor] = None, b2: Optional[torch.Tensor] = None,
                residual: Optional[torch.Tensor] = None, n_per_group: int = 0,
                a2_group_kofs: int = 0, bias: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp64 ``(ref, bound)`` of ``gemm_mx(a, sfa, b, sfb, out, M, N, K, b_mn_major, a2, b2, residual, n_per_group, a2_group_kofs,
    bias)``:

        out[m, n] = Σ_{k < Kpad} A[m, k]·B[n, k]  +  Σ_{j < K2} a2[m, o(n) + j]·b2[n, j]  +  bias[n]  +  residual[m, n]

    with K2 the width of ``b2`` and o(n) = (n // n_per_group)·a2_group_kofs for a grouped LoRA segment (``n_per_group`` > 0),
    else 0 and K2 the width of ``a2``.

    A the decoded ``a [M, Kpad]`` with scales ``sfa`` (rows M); B the decoded ``b [N, Kpad]`` (K-major) or ``b[:Kpad, :N]ᵀ``
    (``b_mn_major``, the weight read for the input gradient), with scales ``sfb`` for rows N, reduction K.  The reduction runs
    over the padded Kpad = K rounded up to 128 (the quantisers write zeros there).  B is a packed weight: its scales are those
    of its 32 x 32 tiles, the same for each 32 rows, and the kernel reads one per 32-row block.  ``bound`` is Σ|terms| for
    :func:`assert_gemm_close` with ``fp8=True``.  An Inf scale or a NaN element makes the outputs it feeds non-finite."""
    Kp = _pad128(K)
    A = mx_decode(a, sfa, M, K)
    bb = b[:Kp, :N].t() if b_mn_major else b[:N, :Kp]
    B = mx_decode(bb, sfb, N, K)
    ref, bound = A @ B.t(), A.abs() @ B.abs().t()
    if a2 is not None and n_per_group > 0:
        k2 = b2.shape[1]
        for n0 in range(0, N, n_per_group):
            n1, o = min(N, n0 + n_per_group), n0 // n_per_group * a2_group_kofs
            x, y = a2[:M, o:o + k2].to(_F64), b2[n0:n1].to(_F64)
            ref[:, n0:n1] += x @ y.t()
            bound[:, n0:n1] += x.abs() @ y.abs().t()
    elif a2 is not None:
        x, y = a2[:M].to(_F64), b2[:N].to(_F64)
        ref, bound = ref + x @ y.t(), bound + x.abs() @ y.abs().t()
    if bias is not None:
        c = bias[:N].to(_F64).unsqueeze(0)
        ref, bound = ref + c, bound + c.abs()
    if residual is not None:
        r = residual[:M, :N].to(_F64)
        ref, bound = ref + r, bound + r.abs()
    return ref, bound


def assert_e4m3_bytes_equal(name: str, got: torch.Tensor, expected: torch.Tensor) -> None:
    """E4M3 bytes equal bit for bit, except that any NaN byte (0x7F / 0xFF) matches any other."""
    nan_g, nan_e = (got & 0x7F) == 0x7F, (expected.to(got.device) & 0x7F) == 0x7F
    same = torch.where(nan_e, nan_g, (got == expected.to(got.device)) & ~nan_g)
    if not bool(same.all()):
        idx = tuple(int(i) for i in (~same).nonzero()[0])
        raise AssertionError(f"{name} differs at {int((~same).sum())} of {got.numel()} bytes; first at {idx}: "
                             f"got 0x{int(got[idx]):02x} expected 0x{int(expected[idx]):02x}")


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
