"""Model-independent machinery of the whole-model fused executors (:mod:`.fused_llama`, :mod:`.fused_pythia`).

An executor subclass owns what depends on the model: its checks of a model's shapes, the order of its trainable parameters and
their stacked views, its own buffers (``_alloc_layers``) and the ``_forward`` / ``_backward`` of one micro-batch.  This module
provides the rest:

* the checks every ``supports`` / ``supports_full_rank`` shares: the ReLoRA wrapper, fp8 in full-rank training, the native
  attention head dim and, last, the device;
* the constructor preamble (sizes, ReLoRA rank / dropout / scale, attention backend, side stream, environment knobs) and the flat
  fp32-gradient parameter store with stacked views; the gradient transport, ``update()`` and the optimizer are those of every
  stepper (:class:`.stepper.Stepper`, ``parallel.grad_sync``);
* the buffers both executors share, the per-layer slot selection, the SDPA fallback attention and the embedding backward;
* ``merge_and_reinit()``, on bf16 weights and on MXFP8-packed ones;
* one CUDA graph per micro-batch shape, capture / replay and launch counting;
* activation checkpointing (``activation_checkpointing=True``): the per-layer buffers shrink to two slots and the backward re-runs
  each lower layer's forward (the executor's ``_layer_fwd``) before that layer's backward (``_recompute``);
* the LoRA group forward / backward on the wgmma GEMM and the fused input-gradient kernel, and the chunked LM head + CE.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F_

from ..ops import fused
from ..parallel.flat import FlatParamStore
from ..parallel.grad_sync import broadcast_params, peer_transport
from ..relora import ReLoRaModel
from .stepper import Stepper

BF = torch.bfloat16


# ---------------------------------------------------------------------- checks shared by every supports() / supports_full_rank()
# Each returns why the executor declines ``model``, or None.
def relora_refusal(model, inner_cls, other_model: str) -> Optional[str]:
    """The ReLoRA wrapper: a ``ReLoRaModel`` around an ``inner_cls`` (else ``other_model``) on the plain recipe."""
    if not isinstance(model, ReLoRaModel):
        return "full-rank training uses the module path"
    if not isinstance(model.wrapped_model, inner_cls):
        return other_model
    if model.lora_only or model.trainable_scaling or model._config.quantize is not None:
        return "lora_only / trainable scaling / quantized frozen weights use the module path"
    return None


def full_rank_refusal(model, cls, other_model: str, args) -> Optional[str]:
    """A bare ``cls`` (else ``other_model``), and no fp8 frozen-weight recipe: full-rank training has no frozen weights."""
    if not isinstance(model, cls):
        return other_model
    if getattr(args, "frozen_dtype", None) in ("fp8", "fp8_full"):
        return f"--frozen_dtype {args.frozen_dtype} has no frozen weights to act on in full-rank training"
    return None


def native_attention_refusal(hd: int, args) -> Optional[str]:
    attention = getattr(args, "attention", "auto")
    if attention == "native" and fused.attention_backend(hd, attention) != "native":
        return f"--attention native supports head_dim <= {fused.NATIVE_ATTENTION_MAX_HEAD_DIM}, got {hd}"
    return None


def checkpointing_refusal(args) -> Optional[str]:
    """Activation checkpointing with the fp8 frozen-weight path: its forward records every site's activation amax, so a recomputed
    layer would record it twice and change the delayed scales of the next step."""
    if getattr(args, "activation_checkpointing", False) and getattr(args, "frozen_dtype", None) in ("fp8", "fp8_full"):
        return (f"--activation_checkpointing cannot be combined with --frozen_dtype {args.frozen_dtype}: the fp8 forward records "
                "activation amax for its delayed scales, and a recomputed layer would record it again")
    return None


def device_refusal(model) -> Optional[str]:
    """Checked after the shapes, so their reasons are visible on a CPU model."""
    p = next(model.parameters())
    return None if p.is_cuda and p.dtype == BF else "needs CUDA + bfloat16"


class LayerViews:
    """Views of one layer's parameters and gradients, None where a mode has no such tensor (the LoRA factors in full-rank training,
    the projection-weight gradients under ReLoRA).  Each executor lists its view names in ``__slots__``, so a misspelt name fails."""

    __slots__ = ()

    def __init__(self):
        for k in self.__slots__:
            setattr(self, k, None)


class FusedStepperBase(Stepper):
    # ------------------------------------------------------------------ construction helpers
    def __init__(self, model, info, supports, supports_full_rank, *, grad_accumulation: int, clip_grad_norm: float,
                 cuda_graphs: bool, ce_chunk: int, overlap_wgrad: bool, attention: str, deterministic: bool,
                 activation_checkpointing: bool = False):
        """Settings and sizes every executor has; ``supports`` / ``supports_full_rank`` are the executor's checks of a ReLoRA model
        and of a bare one (full-rank training).  ``activation_checkpointing``: keep each layer's input (and the wgmma attention's
        output and log-sum-exp) and recompute the rest of a layer in the backward (see ``_recompute``)."""
        self.full = not isinstance(model, ReLoRaModel)
        ok, why = supports_full_rank(model) if self.full else supports(model)
        if not ok:
            raise RuntimeError(why)
        self.model, self.info = model, info
        self.inner = model if self.full else model.wrapped_model
        self.C = fused._C()
        self.ga = grad_accumulation
        self.clip = clip_grad_norm
        self.use_graphs = cuda_graphs
        self.ce_chunk = ce_chunk
        cfg = self.inner.config
        self.h, self.f, self.nh, self.V = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.vocab_size
        self.hd = self.h // self.nh
        self.L = cfg.num_hidden_layers
        self.r = 0 if self.full else model.r
        self.p = 0.0 if self.full else float(model.lora_dropout)
        self.scale = 1.0 if self.full else float(model.lora_alpha) / model.r
        self.device = info.device
        broadcast_params(model)
        attention = os.environ.get("RELORA_B200_ATTENTION", attention)
        # auto: this repo's wgmma kernels (csrc/attention.cu) for head_dim <= 64 -- the hot path then contains no library
        # attention call -- and torch SDPA (cuDNN) above; native: the kernels up to head_dim 256; sdpa: torch SDPA
        # (bench/attn_bench.py times both)
        self.native_attn = fused.attention_backend(self.hd, attention) == "native"
        if attention == "native" and not self.native_attn:
            raise RuntimeError(f"--attention native supports head_dim <= {fused.NATIVE_ATTENTION_MAX_HEAD_DIM} (multiple of 8), "
                               f"got {self.hd}")
        self._attn_saved: Dict[int, tuple] = {}  # SDPA: (o, q, k, v) per layer of the training forward, until its backward
        self.recompute = bool(activation_checkpointing)
        self.side = torch.cuda.Stream(device=self.device) if overlap_wgrad else None
        self.fp8 = self.fp8_bwd = False  # E4M3 frozen weights (csrc/fp8.cu): an executor that has them turns them on
        self.mx = False  # MXFP8-packed frozen stacks (csrc/gemm_mx.cu): likewise
        self.fused_dx = True
        # stacked output width from which the LoRA input gradient uses two kernels (see _lora_group_bwd); 0: the executor's default
        self.dx_split_k = int(os.environ.get("RELORA_B200_DX_SPLIT_K", "0"))
        # --deterministic asks for fixed summation orders; each executor sets which of its GEMMs give up split-K (wgrad_split_k)
        self.deterministic = deterministic or os.environ.get("RELORA_B200_DETERMINISTIC", "0") == "1"
        # embedding backward without atomics (default); RELORA_B200_ATOMIC_EMBEDDING=1 selects the atomicAdd scatter
        self.deterministic_embedding = os.environ.get("RELORA_B200_ATOMIC_EMBEDDING", "0") != "1"

    def _build_store(self, params: List[torch.nn.Parameter], transport: str,
                     padded: Optional[Dict[int, Tuple[int, int]]] = None) -> None:
        """Gradient transport and flat fp32-gradient store over ``params``, which must be every trainable parameter of the model.
        Their order is the store's layout (stacked views, checkpoints, ZeRO shards and the peer-memory update depend on it);
        ``padded`` maps parameters to zero-padded storage shapes."""
        name_of = {id(p): n for n, p in self.model.named_parameters()}
        named = [(name_of[id(p)], p) for p in params]
        seen = {id(p) for p in params}
        extra = [n for n, p in self.model.named_parameters() if p.requires_grad and id(p) not in seen]
        if extra:
            raise RuntimeError(f"unexpected trainable parameters for the fused executor: {extra}")
        self.comm = peer_transport(self.info, transport)
        self.store = FlatParamStore(named, world_size=self.info.world_size, grad_dtype=torch.float32, bind_grads=False,
                                    allocator=self.comm.allocator() if self.comm is not None else None,
                                    storage_shapes=padded or {})

    def _stacked_view(self, p, rows_mult: int = 1, rows: Optional[int] = None):
        """(params, grads) views over ``rows_mult`` adjacent parameters of the flat store, starting at ``p``; or, with ``rows``,
        over adjacent 2-D parameters of ``p``'s width and ``rows`` rows in all (blocks of unequal row counts, such as the LoRA
        B factors of q | k | v under grouped-query attention)."""
        o, n = self.store.segment(p)
        ps = self.store.storage.get(id(p), tuple(p.shape))  # padded block shape where one exists
        if rows is not None:
            return self.store.params[o:o + rows * ps[1]].view(rows, ps[1]), self.store.grads[o:o + rows * ps[1]].view(rows, ps[1])
        shape = (ps[0] * rows_mult, ps[1]) if p.dim() == 2 else (ps[0] * rows_mult,)
        tot = n * rows_mult
        return self.store.params[o:o + tot].view(shape), self.store.grads[o:o + tot].view(shape)

    def _init_optimizer(self, *, lr, betas, eps, weight_decay, zero: bool, native) -> None:
        # fp32 gradients: they cross the wire as a bf16 copy
        self._init_update(zero=zero, stage_bf16=True, native=native or fused.NativeOptim(), lr=lr, betas=betas, eps=eps,
                          weight_decay=weight_decay)
        self.seed = fused.seed_state.get(self.device)
        self._shape = None
        self._graph = None
        self._replays = 0
        self._launches_per_micro = 0
        self._wg_done: Dict[str, torch.cuda.Event] = {}

    # ------------------------------------------------------------------ hooks of the subclasses
    def _alloc_layers(self, B: int, T: int) -> None:
        """The executor's own buffers for a [B, T] micro-batch (``_alloc`` has set ``B_`` / ``T_`` / ``M_`` and ``x_in``); those
        the backward reads per layer have ``n_slots`` slots and are listed in ``self._slotted``."""
        raise NotImplementedError

    def _layer_fwd(self, l: int, S, sl: int, x, x_next, train: bool, recompute: bool = False) -> None:
        """Forward of layer ``l`` from ``x`` into ``x_next``, its saved activations in slot ``sl``.  ``recompute``: the backward's
        re-run of a training layer (see ``_recompute``), which reuses the wgmma attention's saved output and writes no layer output."""
        raise NotImplementedError

    def _before_micro(self) -> None:
        """Runs before a micro-step (outside the CUDA graph)."""

    # ------------------------------------------------------------------ one micro-batch
    def _alloc(self, B: int, T: int) -> None:
        dev, L, h = self.device, self.L, self.h
        M = B * T
        self.B_, self.T_, self.M_ = B, T, M
        self.ids = torch.zeros(B, T, dtype=torch.long, device=dev)
        self.labels = torch.zeros(M, dtype=torch.long, device=dev)
        self.x_in = torch.empty(L + 1, M, h, dtype=BF, device=dev)  # layer inputs, saved for the backward ([0], [1] in evaluation)
        self._alloc_layers(B, T)
        if self.native_attn:
            self.attn_o = torch.empty(L, M, h, dtype=BF, device=dev)
            self.lse = torch.empty(L, B, self.nh, T, dtype=torch.float32, device=dev)
            self.delta = torch.empty(B, self.nh, T, dtype=torch.float32, device=dev)
        ldv = (self.V + 7) // 8 * 8
        self.logits = torch.zeros(min(self.ce_chunk, M), ldv, dtype=BF, device=dev)
        self.loss_sum = torch.zeros(1, dtype=torch.float32, device=dev)
        self.count = torch.zeros(1, dtype=torch.float32, device=dev)
        self.loss_out = torch.zeros((), dtype=torch.float32, device=dev)
        self._shape = (B, T)

    @property
    def n_slots(self) -> int:
        """Slots of the per-layer saved activations: one per layer, or two under activation checkpointing."""
        return min(2, self.L) if self.recompute else self.L

    def _slot(self, l: int) -> int:
        """The slot of layer ``l``'s saved activations in training."""
        return l % 2 if self.recompute else l

    def _kept(self, l: int) -> bool:
        """Whether layer ``l``'s activations are still in their slot when its backward starts: always, or under activation
        checkpointing for the top two layers only (no later forward writes their slots)."""
        return not self.recompute or l >= self.L - 2

    def _layer_slots(self, train: bool):
        """(l, views, slot, x, x_next) per layer of the forward: ``slot`` indexes the per-layer saved activations and ``x`` /
        ``x_next`` are the layer's input and output.  Training keeps every layer's (two alternating slots under activation
        checkpointing); evaluation reuses slot 0 and alternates two residual buffers."""
        for l, S in enumerate(self.layers):
            if train:
                yield l, S, self._slot(l), self.x_in[l], self.x_in[l + 1]
            else:
                yield l, S, 0, self.x_in[l % 2], self.x_in[(l + 1) % 2]

    def _recompute(self, l: int) -> None:
        """Before layer ``l``'s backward under activation checkpointing: re-run its forward from the saved input ``x_in[l]`` into
        slot ``l % 2`` (the top two layers are still there).

        The recompute draws the forward's dropout masks: they hash (seed, key), and the seed advances only after the micro-batch's
        backward.  It writes slot ``l % 2`` and the forward transients, on the main stream, while the side stream still runs layer
        ``l + 1``'s weight gradients; those read slot ``(l + 1) % 2`` and the backward's gradient buffers, never what the recompute
        writes.  The slot's previous owner is layer ``l + 2``: its weight gradients read it, and they are done, because the side
        stream runs in FIFO order and layer ``l + 1``'s backward made the main stream wait for the last group layer ``l + 2`` forked
        (``_join("qkv")``, before its attention backward) -- the executor's call site names its join order."""
        if not self._kept(l):
            self._layer_fwd(l, self.layers[l], self._slot(l), self.x_in[l], self.x_in[l + 1], True, recompute=True)

    def saved_bytes_per_layer(self) -> int:
        """Bytes the training forward keeps for one layer besides its input and the wgmma attention's output: one slot of every
        per-layer buffer and, under SDPA, the kept graph's output and log-sum-exp.  Activation checkpointing keeps ``n_slots``
        slots instead of L (and at most three graphs), so it saves about (L - 2) times this."""
        n = sum(t[0].numel() * t.element_size() for t in self._slotted)
        if not self.native_attn:
            n += self.M_ * self.h * 2 + self.B_ * self.nh * self.T_ * 4
        return n

    def _sdpa(self, q, k, v, train: bool, keep: Optional[int] = None, **kw):
        """Causal torch SDPA over [B, heads, T, head_dim] views (the attention where the wgmma kernels are not used).  In training
        the call runs under autograd, so a forward and its recompute pick the same kernel; ``keep`` (a layer index) keeps the graph
        for ``_sdpa_bwd``.  A kept graph reads its views of ``qkv`` in the backward, so it is kept only while their slot is not
        rewritten."""
        if not train:
            return F_.scaled_dot_product_attention(q, k, v, dropout_p=0.0, is_causal=True, **kw)
        q, k, v = (t.detach().requires_grad_() for t in (q, k, v))
        with torch.enable_grad():
            o = F_.scaled_dot_product_attention(q, k, v, dropout_p=0.0, is_causal=True, **kw)
        if keep is not None:
            self._attn_saved[keep] = (o, q, k, v)
        return o.detach()

    def _sdpa_keep(self, l: int, train: bool, recompute: bool) -> Optional[int]:
        """``keep`` for layer ``l``'s SDPA call: the training forward keeps the graphs of the layers whose slots survive until their
        backward; a recompute keeps its own."""
        return l if train and (recompute or self._kept(l)) else None

    def _sdpa_bwd(self, l: int):
        """(dq, dk, dv) of layer ``l``'s SDPA call for the attention-output gradient in ``dattn``."""
        o, q, k, v = self._attn_saved.pop(l)
        return torch.autograd.grad(o, (q, k, v), self.dattn.view(self.B_, self.T_, self.nh, self.hd).transpose(1, 2))

    def _embedding_bwd_and_join(self, dx, tags) -> None:
        """The embedding gradient from ``dx`` (the gradient of the first layer's input), then the main stream waits for every
        side-stream weight gradient (``tags``, in that order)."""
        if self.deterministic_embedding:
            # stable sort of the token ids (12 K keys) -> one writer per table row, fixed summation order: bit-reproducible
            sorted_ids, perm = torch.sort(self.ids.view(-1), stable=True)
            self.C.embedding_bwd_sorted(sorted_ids, perm, dx, self.gW_emb, self.pad_idx)
        else:
            self.C.embedding_bwd(self.ids.view(-1), dx, self.gW_emb, self.pad_idx)
        for tag in tags:
            self._join(tag)
        self._attn_saved.clear()

    def _micro_body(self) -> None:
        self._set_labels()
        self._forward(True)
        self._loss_and_head_backward(True)
        self._backward()
        self.C.seed_advance(self.seed)

    def _eval_body(self) -> None:
        self._forward(False)
        self._loss_and_head_backward(False)

    # ------------------------------------------------------------------ LoRA groups
    def _lora_group_fwd(self, xn, xd, A, B, W, u, out, *, G, K, Ng, residual=None, site=None, prequant=False, bias=None, Nq=None,
                        mx_ready=False, u_only=False):
        """u = s·xd_g·A_gᵀ (grouped) ; out = [xn | u]·[W | B]ᵀ (+ bias) (+ residual).

        ``u_only`` (a recompute of a layer whose output is saved): u alone, by the same GEMM call as the full forward's.

        ``mx_ready`` (packed stacks): the producer of xn already wrote its MX rows into ``self.xq[K]``.

        ``Nq``: width of the first group when it differs from the other G-1 groups' ``Ng`` (the q | k | v projections of
        grouped-query attention); its output columns and the rest are then two launches into column windows of ``out``.

        fp8 path (``site = (layer, index)``): xn is quantised to E4M3 with the site's delayed scale and multiplied with the E4M3
        copy of W on the kind::f8f6f4 tensor-core path; the bf16 LoRA term shares the accumulator, so u is produced pre-divided
        by the product scale s_x·s_w, which the epilogue multiplies back.

        Full-rank training (``A is None``): out = xn·Wᵀ (+ bias) (+ residual), one launch over the whole stacked group."""
        g, r, M = fused.gemm, self.r, self.M_
        if A is None:
            if not u_only:
                g(xn, W, out, M=M, N=W.shape[0], K1=K, residual=residual, bias=bias)
            return
        drop = self.p > 0 and xd.shape[1] == G * K
        if u_only:
            assert not self.fp8
            g(xd, A, u, M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K if drop else 0, alpha=self.scale)
            return
        if self.mx:
            # packed stack W: xn's E4M3 rows and block scales (the bytes the module path's mx.linear quantises), then
            # out = [xq | u]·[W | B]ᵀ on the block-scaled GEMM, the LoRA segment of group g reading u's columns g·r ..
            xq, sfx = self.xq[K]
            if not mx_ready:
                self.C.mx_quantize_rows(xn, xq, sfx)
            g(xd, A, u, M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K if drop else 0, alpha=self.scale)
            if Nq is not None and Nq != Ng:
                assert residual is None and bias is None and G > 1
                o = self.C.mx_sf_bytes(Nq, K)
                self.C.gemm_mx(xq, sfx, W.q[:Nq], W.sf_fwd[:o], out[:, :Nq], M, Nq, K, False, u[:, :r], B[:Nq])
                self.C.gemm_mx(xq, sfx, W.q[Nq:], W.sf_fwd[o:], out[:, Nq:], M, (G - 1) * Ng, K, False, u[:, r:], B[Nq:], None,
                               Ng if G > 2 else 0, r)
                return
            self.C.gemm_mx(xq, sfx, W.q, W.sf_fwd, out, M, G * Ng, K, False, u, B, residual, Ng if G > 1 else 0, r,
                           *(() if bias is None else (bias,)))
            return
        if self.fp8 and site is not None:
            l, s_i = site
            x8 = self.x8_h if K == self.h else self.x8_f
            if not prequant:  # the producer of xn did not emit the E4M3 copy itself
                self.C.fp8_quantize_act(xn, x8, self.inv_sx[l, s_i:s_i + 1], self.act_state[l, s_i, 1:2])
        if self.fp8 and site is not None and not self._fp8_calibrating:
            g(xd, A, u, M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K if drop else 0, alpha=self.scale,
              alpha_dev=self.alpha_inv[l, s_i:s_i + 1])
            g(x8, self.W8[s_i][l], out, M=M, N=G * Ng, K1=K, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, residual=residual,
              fp8=True, alpha_dev=self.alpha_main[l, s_i:s_i + 1])
            return
        g(xd, A, u, M=M, N=G * r, K1=K, n_per_group=r, a1_group_kofs=K if drop else 0, alpha=self.scale)
        if Nq is not None and Nq != Ng:
            assert residual is None and bias is None and G > 1
            g(xn, W[:Nq], out[:, :Nq], M=M, N=Nq, K1=K, a2=u[:, :r], b2=B[:Nq], K2=r)
            g(xn, W[Nq:], out[:, Nq:], M=M, N=(G - 1) * Ng, K1=K, a2=u[:, r:], b2=B[Nq:], K2=r, n_per_group=Ng, a2_group_kofs=r)
            return
        g(xn, W, out, M=M, N=G * Ng, K1=K, a2=u, b2=B, K2=r, n_per_group=Ng, a2_group_kofs=r, residual=residual, bias=bias)

    def _lora_group_bwd(self, dy, S_B, S_W, S_A, gA, gB, xd, u, keys, *, G, K, Ng, base_out, out, tag, site=None, Nq=None,
                        gW=None):
        """Backward of one stacked LoRA group.  dy [M, G·Ng] -> out [M, K] (grad of the group's input).

        ``Nq`` (see ``_lora_group_fwd``): dy is [M, Nq + (G-1)·Ng]; du and dB then run as two launches each, the first group
        alone and the other G-1 groups together.

        The two weight-gradient GEMMs only read (dy, du, xd, u), so they are forked onto a side stream and fill the
        SMs that the skinny du / parts GEMMs and kernel tails of the main chain leave idle; ``self._wg_done[tag]``
        is the event the main stream waits on before it overwrites one of their inputs (see ``_backward``).

        Full-rank training (``S_A is None``): out = dy·W and gW += dyᵀ·xd (fp32, on the side stream like dA / dB)."""
        C, g, M, r, s = self.C, fused.gemm, self.M_, self.r, self.scale
        if S_A is None:
            N = S_W.shape[0]
            wgrad = lambda: g(dy, xd, gW, M=N, N=K, K1=M, a1_mn=True, b1_mn=True, accumulate=True,  # noqa: E731
                              split_k=self.wgrad_split_k)
            if self.side is not None:
                self._fork_wgrads(tag, wgrad)
            g(dy, S_W, out, M=M, N=K, K1=N, b1_mn=True)
            if self.side is None:
                wgrad()
            return
        du = self.du_bufs[tag]
        split = Nq is not None and Nq != Ng
        width = Nq + (G - 1) * Ng if split else G * Ng
        if split:
            assert G > 1 and not (self.fp8 and site is not None)
            g(dy[:, :Nq], S_B[:Nq], du[:, :r], M=M, N=r, K1=Nq, b1_mn=True, alpha=s)
            g(dy[:, Nq:], S_B[Nq:], du[:, r:], M=M, N=(G - 1) * r, K1=Ng, b1_mn=True, n_per_group=r, a1_group_kofs=Ng,
              b1_group_kofs=Ng, b1_local_n=True, alpha=s)
        else:
            # du_g = s · dy_g · B_g          (B stacked [G·Ng, r], read MN-major; K window g·Ng)
            g(dy, S_B, du, M=M, N=G * r, K1=Ng, b1_mn=True, n_per_group=r, a1_group_kofs=Ng if G > 1 else 0,
              b1_group_kofs=Ng if G > 1 else 0, b1_local_n=True, alpha=s)
        drop = self.p > 0
        shared_x = (not drop) or xd.shape[1] != G * K

        def wgrads():  # fp32, accumulated across micro-batches, split-K over tokens
            g(du, xd, gA, M=G * r, N=K, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=self.wgrad_split_k,
              m_per_group=r if G > 1 else 0, b1_mn_ofs_per_mgroup=0 if shared_x else K)
            if split:
                g(dy[:, :Nq], u[:, :r], gB[:Nq], M=Nq, N=r, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=self.wgrad_split_k)
                g(dy[:, Nq:], u[:, r:], gB[Nq:], M=(G - 1) * Ng, N=r, K1=M, a1_mn=True, b1_mn=True, accumulate=True,
                  split_k=self.wgrad_split_k, m_per_group=Ng, b1_mn_ofs_per_mgroup=r)
                return
            # fp8 path: the saved u is u / (s_x·s_w); the product scale is multiplied back here
            g(dy, u, gB, M=G * Ng, N=r, K1=M, a1_mn=True, b1_mn=True, accumulate=True, split_k=self.wgrad_split_k,
              m_per_group=Ng if G > 1 else 0, b1_mn_ofs_per_mgroup=r if G > 1 else 0,
              alpha_dev=self.alpha_main[site[0], site[1]:site[1] + 1] if (self.fp8 and site is not None) else None)

        if self.side is not None:
            self._fork_wgrads(tag, wgrads)
        if self.mx:
            # packed stack S_W: base = dy·W on the block-scaled GEMM (W's bytes read MN-major with the stack's input-gradient
            # scales), then one pass adds the masked low-rank terms
            sd, ks, pp = (self.seed, list(keys), self.p) if drop else (None, [0] * G, 0.0)
            dq, sfd = self.xq[width]
            C.mx_quantize_rows(dy, dq, sfd)
            C.gemm_mx(dq, sfd, S_W.q, S_W.sf_bwd, base_out, M, K, width, True)
            C.lora_dx(None, None, du, S_A, out, sd, ks, pp, base_out)
        elif self.fused_dx:
            sd, ks, pp = (self.seed, list(keys), self.p) if drop else (None, [0] * G, 0.0)
            if width >= self.dx_split_k:
                # long reductions: the frozen-path product runs on the GEMM, whose TMA-store epilogue overlaps the next
                # tile's k-loop, then one light pass adds the masked low-rank terms
                if self.fp8_bwd and site is not None:
                    # E5M2 copy of the output gradient (delayed scale) x E4M3 copy of Wᵀ on the kind::f8f6f4 path
                    l_, s_i = site
                    dy8 = self.dy8[width]
                    C.fp8_quantize_act(dy, dy8, self._inv_sx2[1, l_, s_i:s_i + 1], self._act_state2[1, l_, s_i, 1:2], True)
                if self.fp8_bwd and site is not None and self._fp8_bwd_calibrated:
                    g(dy8, self.W8T[s_i][l_], base_out, M=M, N=K, K1=G * Ng, fp8=2, alpha_dev=self._alpha_main2[1, l_, s_i:s_i + 1])
                else:
                    g(dy, S_W, base_out, M=M, N=K, K1=width, b1_mn=True)
                C.lora_dx(None, None, du, S_A, out, sd, ks, pp, base_out)
            else:
                # one kernel: out = dy·W + Σ_g keep_g ⊙ (du_g·A_g)/(1-p)  (masked LoRA terms folded into the register accumulator)
                C.lora_dx(dy, S_W, du, S_A, out, sd, ks, pp)
        else:
            # frozen path: base = dy · W     (W stacked [G·Ng, K], read MN-major)
            g(dy, S_W, base_out, M=M, N=K, K1=width, b1_mn=True)
            # low-rank path per group: part_g = du_g · A_g
            parts = self.parts.view(-1)[: M * G * K].view(M, G * K)
            g(du, S_A, parts, M=M, N=G * K, K1=r, b1_mn=True, n_per_group=K, a1_group_kofs=r if G > 1 else 0,
              b1_group_kofs=r if G > 1 else 0, b1_local_n=True)
            if drop:
                C.dropout_combine(base_out, parts, out, self.seed, keys, self.p)
            else:
                torch.add(base_out, parts.view(M, G, K).sum(1) if G > 1 else parts, out=out)
        if self.side is None:
            wgrads()

    def _fork_wgrads(self, tag, wgrads):
        """Runs ``wgrads`` on the side stream after the work issued so far; ``self._wg_done[tag]`` marks its end."""
        fork = torch.cuda.Event()
        fork.record()
        self.side.wait_event(fork)
        with torch.cuda.stream(self.side):
            wgrads()
            done = torch.cuda.Event()
            done.record()
        self._wg_done[tag] = done

    def _join(self, tag):
        """Main stream waits for the side-stream weight gradients tagged ``tag`` (no-op if none are pending)."""
        ev = self._wg_done.pop(tag, None)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def _loss_and_head_backward(self, train: bool):
        """Chunked LM head + CE.  In training also dxf and dW_head (so logits never persist)."""
        C, g, M, h, V = self.C, fused.gemm, self.M_, self.h, self.V
        n_valid = self.B_ * (self.T_ - 1)
        self.loss_sum.zero_()
        self.count.zero_()
        grad_scale = 1.0 / (n_valid * self.ga)
        for s in range(0, M, self.ce_chunk):
            m = min(self.ce_chunk, M - s)
            hc = self.xf[s:s + m]
            lg = self.logits[:m]
            g(hc, self.W_head, lg, M=m, N=V, K1=h)
            C.cross_entropy_fwd_bwd(lg, self.labels[s:s + m], V, grad_scale, -100, self.loss_sum, self.count)
            if train:
                g(lg, self.W_head, self.dxf[s:s + m], M=m, N=h, K1=V, b1_mn=True)
                g(lg, hc, self.gW_head, M=V, N=h, K1=m, a1_mn=True, b1_mn=True, accumulate=True)
        torch.div(self.loss_sum[0], float(n_valid), out=self.loss_out)

    def _set_labels(self):
        self.labels.view(self.B_, self.T_)[:, :-1].copy_(self.ids[:, 1:])
        self.labels.view(self.B_, self.T_)[:, -1].fill_(-100)

    # ------------------------------------------------------------------ public stepper interface
    def _ensure_shape(self, B: int, T: int) -> None:
        if self._shape != (B, T):
            self._alloc(B, T)
            self._graph = None

    @torch.no_grad()
    def micro_step(self, input_ids: torch.Tensor) -> torch.Tensor:
        B, T = input_ids.shape
        self._ensure_shape(B, T)
        self.ids.copy_(input_ids, non_blocking=True)
        self._before_micro()
        if not self.use_graphs:
            self._micro_body()
            return self.loss_out.clone()
        if self._graph is None:
            self._capture()
        else:
            self._graph.replay()
            self._replays += 1
        return self.loss_out.clone()

    def _capture(self):
        # warm-up (allocator, cuBLAS/flash workspaces, tensor-map cache) on a side stream, then capture
        grads_backup = self.store.grads.clone()
        seed_backup = self.seed.clone()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self._micro_body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.store.grads.copy_(grads_backup)
        self.seed.copy_(seed_backup)
        n0 = self.C.launch_count()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._micro_body()
        self._launches_per_micro = self.C.launch_count() - n0
        # capture does not execute: run the captured work once for this micro-batch
        self.store.grads.copy_(grads_backup)
        self.seed.copy_(seed_backup)
        del grads_backup
        graph.replay()
        self._replays += 1
        self._graph = graph

    @torch.no_grad()
    def eval_loss(self, input_ids: torch.Tensor) -> torch.Tensor:
        B, T = input_ids.shape
        self._ensure_shape(B, T)
        self.ids.copy_(input_ids)
        self._set_labels()
        self._eval_body()
        return self.loss_out.clone()

    @torch.no_grad()
    def merge_and_reinit(self):
        """W += s·B@A for every module of every layer and its (B, A, W) block (``mods`` / ``merge`` of the layer views; wgmma GEMM
        accumulating into W in fp32), then the hash re-init of the module path: A ~ U(±1/√in) keyed by (seed, restart, module
        index), B = 0.  Packed weights: see ``_merge_packed``."""
        if self.full:
            raise RuntimeError("merge_and_reinit needs a ReLoRA model; full-rank training has no low-rank factors")
        if self.mx:
            self._merge_packed()
            return
        g, r = fused.gemm, self.r
        for S in self.layers:
            for m, (Bm, Am, Wm) in zip(S.mods, S.merge):
                g(Bm, Am, Wm, M=Wm.shape[0], N=Wm.shape[1], K1=r, b1_mn=True, alpha=self.scale, accumulate=True)
                self._reinit_lora(m)
        self.model.n_restarts += 1

    @torch.no_grad()
    def _merge_packed(self) -> None:
        """The merge on MXFP8-packed weights: for each packed weight ``self.Wmx[l][i]`` of a layer, the fp32 delta s·B·A of its
        blocks ``S.merge[i]`` ((B, A, first row) each) on the GEMM, then every 32 x 32 tile requantised in place (``ops/mx.merge_``'s
        contract); then ``_packed_merged(l)`` and the re-init of the layer's modules.  The delta scratch is the size of the
        largest packed weight of a layer and is released afterwards."""
        g, r = fused.gemm, self.r
        delta = torch.empty(max(st.N * st.K for st in self.Wmx[0]), dtype=torch.float32, device=self.device)
        for l, S in enumerate(self.layers):
            for st, blocks in zip(self.Wmx[l], S.merge):
                d = delta[:st.N * st.K].view(st.N, st.K).zero_()
                for Bm, Am, r0 in blocks:
                    g(Bm, Am, d[r0:r0 + Bm.shape[0]], M=Bm.shape[0], N=st.K, K1=r, b1_mn=True, alpha=self.scale, accumulate=True)
                self.C.mx_quantize_weight_2d(None, d, st.q, st.sf_fwd, st.sf_bwd, st.N, st.K)
            self._packed_merged(l)
            for m in S.mods:
                self._reinit_lora(m)
        del delta
        self.model.n_restarts += 1

    def _packed_merged(self, l: int) -> None:
        """Runs after layer ``l``'s packed weights were requantised (an executor whose modules keep copies of them refreshes those)."""

    def _reinit_lora(self, m) -> None:
        """The module path's re-init of one module after its merge: A ~ U(±1/√in) keyed by (seed, restart, module index), B = 0."""
        from ..ops import reference as ref

        sd = ref.mix_seed(self.model.seed, self.model.n_restarts, m.module_index)
        self.C.fill_uniform_hash(m.lora_A.weight.data, sd, 1.0 / math.sqrt(m.in_features))
        m.lora_B.weight.data.zero_()

    def launches_in_window(self, n_steps: int) -> int:
        """Kernel launches of this extension since ``reset_launch_count`` (graph replays included)."""
        return int(self.C.launch_count() + self._replays_since_reset() * self._launches_per_micro)

    def _replays_since_reset(self) -> int:
        return self._replays - getattr(self, "_replay_mark", 0)

    def mark_launch_window(self):
        self._replay_mark = self._replays
        self.C.reset_launch_count()
