"""Python face of the native sm_90a kernels: thin wrappers + autograd functions.

Everything here requires the in-tree extension (``relora_b200/_C.so``); :mod:`.dispatch` decides
when these are used.  Numerics oracles live in :mod:`.reference`.
"""
from __future__ import annotations

import math
import os
from typing import List, Optional, Sequence

import torch

from . import native
from . import reference as ref

_BF16 = torch.bfloat16


def _C():
    return native.require()


# ----------------------------------------------------------------------------- global dropout stream
class _SeedState:
    """Device-resident base seed shared by all dropout-bearing kernels of one micro-step.

    It lives on the device (and is advanced by a one-thread kernel) so that CUDA-graph replays draw
    fresh masks each time without re-capturing.
    """

    def __init__(self):
        self.tensors = {}

    def get(self, device) -> torch.Tensor:
        key = (device.type, device.index)
        t = self.tensors.get(key)
        if t is None:
            t = torch.tensor([0x1234567], dtype=torch.int32, device=device)
            self.tensors[key] = t
        return t

    def set(self, device, value: int) -> None:
        v = int(value) & 0xFFFFFFFF
        if v >= 1 << 31:
            v -= 1 << 32
        self.get(device).fill_(v)

    def advance(self, device) -> None:
        _C().seed_advance(self.get(device))


seed_state = _SeedState()


def seed_value(device) -> int:
    return int(seed_state.get(device).item()) & 0xFFFFFFFF


# ----------------------------------------------------------------------------- GEMM
def gemm(
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
    out_dtype: torch.dtype = _BF16,
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
) -> torch.Tensor:
    """``out[M,N] = alpha·(a1·b1ᵀ + a2·b2ᵀ) (+ residual) (+ out)`` on the wgmma kernel.

    ``block_n``: output tile width, 0 = the dispatcher's wave-count rule (``gemm_block_n``), else 128, 192 or 256.
    ``pair``: CTA pairs, two M tiles of one N tile sharing each B tile through TMA multicast: -1 lets the dispatcher
    choose (``gemm_pairs``), 0 turns them off, 1 asks for them where the call form allows (the 256-wide tile does not).
    ``fp8``: 1 = ``a1`` / ``b1`` hold E4M3 bytes (K-major), 2 = ``a1`` is E5M2 (gradients); ``alpha_dev``: fp32 device scalar multiplied into ``alpha``.

    K-major operands are ``[rows, K]`` row-major; with ``a1_mn`` / ``b1_mn`` the tensor is
    ``[K, rows]`` row-major (the natural layout of activations for weight-gradient GEMMs).
    """
    if M is None:
        M = a1.shape[1] if a1_mn else a1.shape[0]
    if K1 is None:
        K1 = a1.shape[0] if a1_mn else a1.shape[1]
    if N is None:
        N = b1.shape[1] if b1_mn else b1.shape[0]
    if a2 is not None and K2 == 0:
        K2 = b2.shape[1]
    if out is None:
        ld = (N + 7) // 8 * 8
        buf = torch.empty(M, ld, dtype=out_dtype, device=a1.device)
        out = buf[:, :N] if ld != N else buf
        assert not accumulate
    _C().gemm(a1, b1, out, M, N, K1, a2, b2, K2, a1_mn, b1_mn, n_per_group, a1_group_kofs, a2_group_kofs,
              residual, float(alpha), accumulate, block_n, split_k, b1_group_kofs, b1_local_n, m_per_group,
              b1_mn_ofs_per_mgroup, bias, pair, int(fp8), alpha_dev)
    return out


# ----------------------------------------------------------------------------- RMSNorm
_norm_ws = {}


def norm_workspace(device, H: int):
    """(fp32 workspace, int32 ticket) for the warp-per-row RMSNorm backward (shared by all layers of a device)."""
    key = (device.type, device.index)
    cur = _norm_ws.get(key)
    need = _C().rmsnorm_bwd_ws_blocks() * H
    if cur is None or cur[0].numel() < need:
        cur = (torch.empty(need, dtype=torch.float32, device=device), torch.zeros(1, dtype=torch.int32, device=device))
        _norm_ws[key] = cur
    return cur


class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        xc = x.contiguous()
        y = torch.empty_like(xc)
        rstd = torch.empty(xc.numel() // xc.shape[-1], dtype=torch.float32, device=x.device)
        _C().rmsnorm_fwd(xc, weight.contiguous(), y, rstd, eps, None, None, [], 0.0)
        ctx.save_for_backward(xc, weight, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, rstd = ctx.saved_tensors
        dx = torch.empty_like(x)
        dw = torch.zeros(weight.shape, dtype=torch.float32, device=x.device)
        ws, tk = norm_workspace(x.device, x.shape[-1])
        _C().rmsnorm_bwd(dy.contiguous(), x, weight.contiguous(), rstd, None, dx, dw, ws, tk)
        return dx, dw.to(weight.dtype), None


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    return _RMSNormFn.apply(x, weight, eps)


# ----------------------------------------------------------------------------- GPT-NeoX / Pythia leaf ops (csrc/neox.cu)
class _LayerNormFn(torch.autograd.Function):
    """``nn.LayerNorm`` with affine weight / bias (reference modeling_pythia.py:413-414) on the warp-per-row kernels."""

    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1]).contiguous()
        y = torch.empty_like(x2)
        mean = torch.empty(x2.shape[0], dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        _C().layernorm_fwd(x2, weight.contiguous(), None if bias is None else bias.contiguous(), y, mean, rstd, float(eps))
        ctx.save_for_backward(x2, weight, mean, rstd)
        ctx.has_bias = bias is not None
        ctx.shape = shp
        return y.view(shp)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, mean, rstd = ctx.saved_tensors
        dy2 = dy.reshape(x2.shape).contiguous()
        dx = torch.empty_like(x2)
        dw = torch.zeros(x2.shape[1], dtype=torch.float32, device=x2.device)
        db = torch.zeros_like(dw) if ctx.has_bias else None
        _C().layernorm_bwd(dy2, x2, weight.contiguous(), mean, rstd, dx, dw, db)
        return dx.view(ctx.shape), dw.to(weight.dtype), (db.to(weight.dtype) if db is not None else None), None


def layernorm_supported(x: torch.Tensor) -> bool:
    return x.is_cuda and x.dtype == _BF16 and x.shape[-1] % 8 == 0 and x.shape[-1] <= 2048


def layernorm(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], eps: float) -> torch.Tensor:
    return _LayerNormFn.apply(x, weight, bias, eps)


class _GeluFn(torch.autograd.Function):
    """Exact (erf) or tanh GELU (reference modeling_pythia.py:395-406); the backward recomputes the derivative from the input."""

    @staticmethod
    def forward(ctx, z, tanh_approx):
        zc = z.contiguous()
        a = torch.empty_like(zc)
        _C().gelu_fwd(zc, a, bool(tanh_approx))
        ctx.save_for_backward(zc)
        ctx.tanh_approx = bool(tanh_approx)
        return a

    @staticmethod
    def backward(ctx, da):
        (z,) = ctx.saved_tensors
        dz = torch.empty_like(z)
        _C().gelu_bwd(da.contiguous(), z, dz, ctx.tanh_approx)
        return dz, None


def gelu(z: torch.Tensor, tanh_approx: bool = False) -> torch.Tensor:
    return _GeluFn.apply(z, tanh_approx)


class _NeoXRopeFn(torch.autograd.Function):
    """Partial rotary embedding on the fused ``query_key_value`` output ``[B, T, nh, 3*hd]`` (reference modeling_pythia.py:172-197):
    the first ``rot`` dims of q and k of every head are rotated with fp32 tables; backward applies the inverse rotation."""

    @staticmethod
    def forward(ctx, qkv, cos, sin, nh, hd, rot):
        B, T = qkv.shape[0], qkv.shape[1]
        out = qkv.reshape(B * T, nh * 3 * hd).clone()
        _C().neox_rope(out, T, nh, hd, rot, cos, sin, 0, False)
        ctx.save_for_backward(cos, sin)
        ctx.meta = (B, T, nh, hd, rot, qkv.shape)
        return out.view(qkv.shape)

    @staticmethod
    def backward(ctx, g):
        cos, sin = ctx.saved_tensors
        B, T, nh, hd, rot, shp = ctx.meta
        gg = g.reshape(B * T, nh * 3 * hd).clone()
        _C().neox_rope(gg, T, nh, hd, rot, cos, sin, 0, True)
        return gg.view(shp), None, None, None, None, None


def neox_rope(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, nh: int, hd: int, rot: int) -> torch.Tensor:
    return _NeoXRopeFn.apply(qkv, cos, sin, nh, hd, rot)


# ----------------------------------------------------------------------------- LoRA linear (module path)
class _LoRALinearFn(torch.autograd.Function):
    """y = x Wᵀ + s·drop(x) Aᵀ Bᵀ with the low-rank up-projection folded into the frozen GEMM's K loop.

    forward  : xd = mask⊙x/(1-p);  u = s·xd·Aᵀ;  y = [x | u]·[W | B]ᵀ                (3 kernels)
    backward : du = s·dy·B;  dx = dy·W + mask⊙(du·A)/(1-p);  dA = duᵀ·xd;  dB = dyᵀ·u
    (reference: relora.py:309-323 — F.linear, dropout, two linears, mul, in-place add)
    """

    @staticmethod
    def forward(ctx, x, weight, lora_a, lora_b, scale, p, key, training, bias=None):
        C = _C()
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        M, K = x2.shape
        N, r = lora_b.shape
        drop = training and p > 0.0
        seed = seed_state.get(x.device)
        if drop:
            xd = torch.empty(M, K, dtype=_BF16, device=x.device)
            C.dropout_expand(x2, xd, seed, [key], p)
        else:
            xd = x2
        u = gemm(xd, lora_a, alpha=scale)  # [M, r]
        y = gemm(x2, weight, a2=u, b2=lora_b, K2=r, bias=bias)  # bias (Pythia) is added in the GEMM epilogue
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x2, weight, lora_a, lora_b, u)
        ctx.meta = (scale, p if drop else 0.0, key, shp)
        # the seed tensor is advanced once per micro-step *after* backward, so backward re-derives the mask
        return y.reshape(*shp[:-1], N)

    @staticmethod
    def backward(ctx, dy):
        C = _C()
        x2, weight, lora_a, lora_b, u = ctx.saved_tensors
        scale, p, key, shp = ctx.meta
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        M, K = x2.shape
        N, r = lora_b.shape
        seed = seed_state.get(x2.device)
        # du = s · dy · B       (B operand = Bᵀ, read MN-major straight from lora_B [N, r])
        du = gemm(dy2, lora_b, M=M, N=r, K1=N, b1_mn=True, alpha=scale)
        # dx = dy · W            (W [N, K] read MN-major)
        dx = gemm(dy2, weight, M=M, N=K, K1=N, b1_mn=True)
        dxl = gemm(du, lora_a, M=M, N=K, K1=r, b1_mn=True)
        if p > 0.0:
            out = torch.empty_like(dx)
            C.dropout_combine(dx, dxl.reshape(1, M, K), out, seed, [key], p)
            dx = out
            xd = torch.empty(M, K, dtype=_BF16, device=x2.device)
            C.dropout_expand(x2, xd, seed, [key], p)
        else:
            dx = dx + dxl
            xd = x2
        # weight gradients: reductions over the token dimension, both operands read MN-major, split-K
        da = torch.zeros(r, K, dtype=torch.float32, device=x2.device)
        gemm(du, xd, da, M=r, N=K, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=0)
        db = torch.zeros(N, r, dtype=torch.float32, device=x2.device)
        # u already carries the factor s (u = s·xd·Aᵀ), and dB = s·dyᵀ·(xd·Aᵀ) = dyᵀ·u
        gemm(dy2, u, db, M=N, N=r, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=0)
        dbias = dy2.float().sum(0).to(dy2.dtype) if ctx.has_bias else None
        return dx.reshape(shp), None, da.to(lora_a.dtype), db.to(lora_b.dtype), None, None, None, None, dbias


def relora_linear_module(module, x: torch.Tensor) -> torch.Tensor:
    """Fused forward for a :class:`ReLoRaLinear` (falls back to PyTorch for the unsupported corners)."""
    unsupported = (
        module.lora_only or module.trainable_scaling or module.quantize is not None
        or module.in_features % 8 or module.out_features % 8 or module.r % 8
    )
    if unsupported:
        import torch.nn.functional as F

        if module.lora_only:
            return module.lora_B(module.lora_A(module.lora_dropout(x))) * module._post_lora_scale()
        if module.quantize is not None:
            from ..relora.linear import packed_linear

            out = packed_linear(x, module.qweight, module.bias)  # only the packed bytes are resident
        else:
            out = F.linear(x, module.weight, module.bias)
        pd = float(module.lora_dropout.p) if module.training else 0.0
        xd = x
        if pd > 0.0 and x.is_cuda:
            # same counter-based mask as the kernels (shapes the TMA path cannot take, e.g. llama_1b's 5461-wide MLP)
            from . import reference as ref

            base = int(seed_state.get(x.device).item()) & 0xFFFFFFFF
            x2 = x.reshape(-1, x.shape[-1])
            keep = ref.dropout_keep_mask(ref.mix_seed(base, int(module.module_index) + 1), x2.shape[0], x2.shape[1], pd, device=x.device)
            xd = (x2 * keep.to(x.dtype) * (1.0 / (1.0 - pd))).reshape(x.shape).to(x.dtype)
        elif pd > 0.0:
            xd = module.lora_dropout(x)
        return out + module.lora_B(module.lora_A(xd)) * module._post_lora_scale()
    return _LoRALinearFn.apply(x, module.weight, module.lora_A.weight, module.lora_B.weight, float(module.scaling),
                               float(module.lora_dropout.p), int(module.module_index) + 1, module.training, module.bias)


# ----------------------------------------------------------------------------- causal attention (module path)
NATIVE_ATTENTION_MAX_HEAD_DIM = 256  # what the wgmma kernels (csrc/attention.cu) accept
AUTO_ATTENTION_MAX_HEAD_DIM = 64     # where `--attention auto` uses them


def attention_backend(head_dim: int, mode: Optional[str] = None, q: Optional[torch.Tensor] = None) -> str:
    """Which causal-attention implementation runs: ``"native"`` (the wgmma kernels of csrc/attention.cu) or ``"sdpa"``
    (torch SDPA, cuDNN).  ``mode`` is the ``--attention`` choice; by default ``RELORA_B200_ATTENTION``, else ``auto``.

    * ``sdpa``: always SDPA.
    * ``auto``: native for ``head_dim % 8 == 0 and head_dim <= 64``, SDPA otherwise.
    * ``native``: native for ``head_dim % 8 == 0 and head_dim <= 256``, SDPA otherwise (the fused executor raises there).

    With ``q`` given, native also needs q on CUDA in bf16."""
    mode = mode or os.environ.get("RELORA_B200_ATTENTION", "auto")
    if mode not in ("auto", "native", "sdpa"):
        raise ValueError(f"attention mode must be auto, native or sdpa, got {mode!r}")
    if mode == "sdpa" or (q is not None and not (q.is_cuda and q.dtype == _BF16)):
        return "sdpa"
    limit = NATIVE_ATTENTION_MAX_HEAD_DIM if mode == "native" else AUTO_ATTENTION_MAX_HEAD_DIM
    return "native" if head_dim % 8 == 0 and 0 < head_dim <= limit else "sdpa"


class _CausalAttentionFn(torch.autograd.Function):
    """Causal self-attention on the wgmma kernels for ``q, k, v [B, nh, T, hd]`` (RoPE already applied).

    The kernels read a packed ``[B*T, 3*nh*hd]`` projection buffer in place (that is what the fused executor hands them);
    the module path packs its three projection outputs once.  Replaces ``F.scaled_dot_product_attention(is_causal=True)``
    (reference modeling_llama.py:222-224)."""

    @staticmethod
    def forward(ctx, q, k, v, scale):
        C = _C()
        B, nh, T, hd = q.shape
        M, h = B * T, nh * hd
        qkv = torch.empty(M, 3 * h, dtype=_BF16, device=q.device)
        q5 = qkv.view(B, T, 3, nh, hd)
        q5[:, :, 0].copy_(q.transpose(1, 2))
        q5[:, :, 1].copy_(k.transpose(1, 2))
        q5[:, :, 2].copy_(v.transpose(1, 2))
        out = torch.empty(M, h, dtype=_BF16, device=q.device)
        lse = torch.empty(B, nh, T, dtype=torch.float32, device=q.device)
        C.attention_fwd(qkv, out, lse, B, T, nh, hd, float(scale))
        ctx.save_for_backward(qkv, out, lse)
        ctx.meta = (B, nh, T, hd, float(scale))
        return out.view(B, T, nh, hd).transpose(1, 2)

    @staticmethod
    def backward(ctx, dout):
        C = _C()
        qkv, out, lse = ctx.saved_tensors
        B, nh, T, hd, scale = ctx.meta
        M, h = B * T, nh * hd
        do = dout.transpose(1, 2).reshape(M, h)
        if not do.is_contiguous():
            do = do.contiguous()
        dqkv = torch.empty_like(qkv)
        delta = torch.empty(B, nh, T, dtype=torch.float32, device=qkv.device)
        C.attention_bwd(qkv, out, do, lse, delta, dqkv, B, T, nh, hd, scale)
        d5 = dqkv.view(B, T, 3, nh, hd)
        return d5[:, :, 0].transpose(1, 2), d5[:, :, 1].transpose(1, 2), d5[:, :, 2].transpose(1, 2), None


def causal_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: Optional[float] = None) -> torch.Tensor:
    hd = q.shape[-1]
    return _CausalAttentionFn.apply(q, k, v, (1.0 / math.sqrt(hd)) if scale is None else scale)


# ----------------------------------------------------------------------------- LM head + cross entropy
class _LMHeadCEFn(torch.autograd.Function):
    """Chunked LM-head GEMM + softmax-CE; forward also produces dh and dW (Liger-style), so the
    ``[tokens, V]`` logits never exist in full and backward is a scale."""

    @staticmethod
    def forward(ctx, h, w_head, labels, chunk):
        C = _C()
        B, T, H = h.shape
        V = w_head.shape[0]
        hs = h[:, :-1].reshape(-1, H)
        tgt = labels[:, 1:].reshape(-1).contiguous()
        n = hs.shape[0]
        ldv = (V + 7) // 8 * 8
        loss_sum = torch.zeros(1, dtype=torch.float32, device=h.device)
        count = torch.zeros(1, dtype=torch.float32, device=h.device)
        dhs = torch.empty(n, H, dtype=_BF16, device=h.device)
        dw = torch.zeros(V, H, dtype=torch.float32, device=h.device)
        # mean over valid tokens: scale gradients by 1/count afterwards (count known only after the pass)
        logits_buf = torch.empty(min(chunk, n), ldv, dtype=_BF16, device=h.device)
        for s in range(0, n, chunk):
            m = min(chunk, n - s)
            hc = hs[s : s + m].contiguous()
            lg = logits_buf[:m]
            gemm(hc, w_head, lg, M=m, N=V, K1=H)
            C.cross_entropy_fwd_bwd(lg, tgt[s : s + m], V, 1.0, -100, loss_sum, count)
            # dh = dlogits · W   (W [V, H] read MN-major);  dW += dlogitsᵀ · h
            gemm(lg, w_head, dhs[s : s + m], M=m, N=H, K1=V, b1_mn=True)
            gemm(lg, hc, dw, M=V, N=H, K1=m, a1_mn=True, b1_mn=True, accumulate=True)
        inv = 1.0 / count.clamp(min=1.0)
        loss = (loss_sum * inv).reshape(())
        ctx.save_for_backward(dhs, dw, inv)
        ctx.shape = (B, T, H)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        dhs, dw, inv = ctx.saved_tensors
        B, T, H = ctx.shape
        g = (dloss.float() * inv).reshape(())
        dh = torch.zeros(B, T, H, dtype=_BF16, device=dhs.device)
        dh[:, :-1] = (dhs.float() * g).to(_BF16).view(B, T - 1, H)
        return dh, (dw * g).to(_BF16), None, None


def lm_head_cross_entropy(h: torch.Tensor, w_head: torch.Tensor, labels: torch.Tensor, chunk: int = 4096) -> torch.Tensor:
    return _LMHeadCEFn.apply(h, w_head, labels, chunk)


# ----------------------------------------------------------------------------- merge / re-init
@torch.no_grad()
def merge_and_reinit_modules(modules: Sequence, *, seed: int, restart_index: int) -> bool:
    """``W += s·B@A`` (wgmma GEMM accumulating into W in fp32, one rounding) + hash-based kaiming
    re-init of A + zeroing of B, for a list of :class:`ReLoRaLinear`.  Reference: relora.py:269-307."""
    C = _C()
    for m in modules:
        if m.lora_only or m.quantize is not None or m.trainable_scaling or m.in_features % 8 or m.out_features % 8 or m.r % 8:
            return False
    for m in modules:
        w = m.weight.data  # [N, K]
        # W[N,K] += s · B[N,r] · A[r,K]:  A-operand = lora_B (K-major over r), B-operand = lora_A read MN-major
        gemm(m.lora_B.weight.data, m.lora_A.weight.data, w, M=m.out_features, N=m.in_features, K1=m.r, b1_mn=True,
             alpha=float(m.scaling), accumulate=True)
        s = ref.mix_seed(seed, restart_index, m.module_index)
        C.fill_uniform_hash(m.lora_A.weight.data, s, 1.0 / math.sqrt(m.in_features))
        m.lora_B.weight.data.zero_()
    return True


# ----------------------------------------------------------------------------- optimizer kernels
class NativeOptim:
    """Adapter handed to :class:`relora_b200.parallel.flat.FlatAdamW` (``native=``)."""

    def __init__(self):
        self._ws = {}

    def adamw_flat(self, p, g, m, v, lr, b1, b2, eps, wd, step, grad_scale, skip, step_dev=None):
        gs_t, gs_h = (grad_scale, 1.0) if torch.is_tensor(grad_scale) else (None, float(grad_scale))
        if gs_t is not None:
            gs_t = gs_t.reshape(1).float()
        sk = None
        if skip is not None:
            sk = skip.reshape(1).float() if torch.is_tensor(skip) else torch.tensor([float(skip)], device=p.device)
        _C().adamw_flat(p, g, m, v, lr, b1, b2, eps, wd, step, gs_t, gs_h, sk, None if step_dev is None else step_dev.reshape(1))

    def random_prune_(self, seg, ratio, seed, col_offset):
        _C().random_prune(seg, ratio, seed, col_offset)

    def magnitude_prune_(self, seg, ratio):
        dev = seg.device
        ws = self._ws.get(dev)
        if ws is None:
            ws = (torch.empty(_C().quantile_workspace_bytes(), dtype=torch.uint8, device=dev),
                  torch.zeros(1, dtype=torch.float32, device=dev))
            self._ws[dev] = ws
        _C().magnitude_prune(seg, ratio, ws[0], ws[1])

    def sumsq(self, x):
        out = torch.zeros(1, dtype=torch.float32, device=x.device)
        _C().sumsq(x, out)
        return out
