"""Whole-model fused executor for Pythia (GPT-NeoX) + ReLoRA on H100.

The Llama executor's design (:mod:`.fused_llama`) applied to the GPT-NeoX block:

* every projection is ONE wgmma GEMM with the LoRA up-projection folded into the K loop and the bias (and, for ``dense`` and
  ``dense_4h_to_h``, the residual) added in the epilogue: ``y = [x | s·xd·Aᵀ]·[W | B]ᵀ + b (+ residual)``;
* one LayerNorm pass writes ``LN1(x)`` and, under parallel residual, ``LN2(x)`` from shared fp32 statistics, each with its LoRA-
  dropout copy; the backward forms ``dx = dres + LN1ᵀ(dy1) + LN2ᵀ(dy2)`` in one pass together with the γ / β gradients and the
  bias gradient of the projections whose output gradient ``dres`` is;
* GELU writes the dropout copy of its output, its backward the bias gradient of ``dense_h_to_4h``; a column sum of ``dqkv`` is the
  ``query_key_value`` bias gradient;
* attention runs on the head-interleaved ``query_key_value`` output in place (wgmma kernels, or SDPA on strided views);
* chunked LM head + CE, one flat fp32 gradient buffer, one CUDA graph per micro-batch (dropout seeds on the device).

The frozen weights stay where the modules keep them; the trainable parameters (LoRA factors, biases, LayerNorms, embeddings) are
views of the flat store, so checkpoints keep the HF GPT-NeoX keys.  Numerics tests compare this executor with the module path on
identical weights and dropout masks.

Full-rank training (a bare ``GPTNeoXForCausalLM``, ``--engine fused``) runs the same layer loop without the low-rank branch: the
four projection weights of each layer are trainable views of the flat store, every projection is one GEMM with the bias (and
residual) epilogue, the input gradient is ``dy·W``, and the fp32 weight gradient ``gW += dyᵀ·x`` runs on the side stream where
``dA`` / ``dB`` run under ReLoRA.  ``x`` is what the executor already saves with p = 0: the norm outputs, the attention output and
the GELU output.

MXFP8-packed frozen weights (``--quantize 8bit``, ``quantize="mxfp8"``): each projection's frozen operand is the module's own packed
weight (``qweight``, an ``ops/mx.MxWeight``; ``query_key_value`` is already one module, so nothing is stacked), the only resident
copy.  Every projection quantises its input to MX rows (``mx_quantize_rows``) and runs ``[xq | u]·[W | B]ᵀ + b (+ residual)`` on
the block-scaled GEMM with the bias in its epilogue.  The backward quantises each output gradient and reads the packed bytes
MN-major; the merge requantises each module's bytes in place.

Parallel residual:   x_next = x + dense(attn(LN1 x)) + b_o + mlp(LN2 x) + b_4
Sequential residual: x1 = x + dense(attn(LN1 x)) + b_o ;  x_next = x1 + mlp(LN2 x1) + b_4
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from ..models.pythia import GPTNeoXForCausalLM
from ..ops import mx
from ..ops.quant import canonical_format
from ..parallel.dist import DistInfo
from ..relora import ReLoRaModel
from .fused_common import (FusedStepperBase, LayerViews, device_refusal, full_rank_refusal, native_attention_refusal,
                           relora_refusal)

BF = torch.bfloat16
MAX_HIDDEN = 2048  # the executor LayerNorm backward keeps its block partials of five [H] vectors in 48 KB of shared memory


def _neox_refusal(model, r=None) -> Optional[str]:
    """Why the executor declines the GPT-NeoX ``model`` (LoRA rank ``r``; None in full-rank training) for its configuration, or
    None."""
    cfg = model.config
    if float(getattr(cfg, "hidden_dropout", 0.0)) != 0.0 or float(getattr(cfg, "attention_dropout", 0.0)) != 0.0:
        return "hidden / attention dropout must be 0"
    layer0 = model.gpt_neox.layers[0]
    if not isinstance(layer0.mlp.act, nn.GELU):
        return "only the GELU activation is fused"
    h, f, nh = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads
    if r is None and (h % 128 or f % 128):
        return f"hidden ({h}) and intermediate ({f}) must be multiples of 128"
    if r is not None and (h % 128 or r % 128 or f % 128):
        return f"hidden ({h}), intermediate ({f}) and rank ({r}) must be multiples of 128"
    if h > MAX_HIDDEN:
        return f"hidden ({h}) must be <= {MAX_HIDDEN} (LayerNorm kernel limit)"
    hd = h // nh
    if hd % 8:
        return f"head_dim ({hd}) must be a multiple of 8 for the attention and rotary kernels"
    if layer0.attention.rotary_ndims % 2:
        return "the number of rotary dims must be even"
    at, mlp = layer0.attention, layer0.mlp
    if any(m.bias is None for m in (at.query_key_value, at.dense, mlp.dense_h_to_4h, mlp.dense_4h_to_h)):
        return "projections without bias use the module path"
    return None


def supports(model, args=None) -> Tuple[bool, str]:
    """(True, "ok") when the Pythia executor can train ``model``, else (False, why)."""
    why = relora_refusal(model, GPTNeoXForCausalLM, "not a GPT-NeoX (Pythia) model")
    if why is None and getattr(args, "frozen_dtype", None) in ("fp8", "fp8_full"):
        why = "fp8 frozen weights are not supported for Pythia"
    why = why or _neox_refusal(model.wrapped_model, model.r) or device_refusal(model.wrapped_model)
    return (False, why) if why else (True, "ok")


def supports_quantized(model, args=None) -> Tuple[bool, str]:
    """Whether the executor can train ``model`` with MXFP8-packed frozen weights (``--engine fused --quantize 8bit``), and if
    not, why.  ``--engine auto`` does not ask: it keeps quantised models on the module path."""
    if not isinstance(model, ReLoRaModel):
        return False, "quantized frozen weights need a ReLoRA model; full-rank training has no frozen weights"
    if not isinstance(model.wrapped_model, GPTNeoXForCausalLM):
        return False, "not a GPT-NeoX (Pythia) model"
    fmt = canonical_format(model._config.quantize)
    if fmt is None:
        return False, "the model's frozen weights are not quantized"
    if fmt != "mxfp8":
        return False, (f"--quantize {model._config.quantize}: only 8bit (mxfp8) frozen weights run on the fused executor; "
                       "4bit (nvfp4) uses --engine module")
    if getattr(args, "frozen_dtype", None) in ("fp8", "fp8_full"):
        return False, f"--frozen_dtype {args.frozen_dtype} cannot be combined with --quantize: the frozen weights are already MXFP8"
    if model.lora_only or model.trainable_scaling:
        return False, "lora_only / trainable scaling with quantized frozen weights use --engine module"
    why = _neox_refusal(model.wrapped_model, model.r) or device_refusal(model.wrapped_model)
    return (False, why) if why else (True, "ok")


def supports_full_rank(model, args=None) -> Tuple[bool, str]:
    """Whether the executor can train ``model`` (an unwrapped GPT-NeoX) full-rank, and if not, why."""
    why = full_rank_refusal(model, GPTNeoXForCausalLM, "only GPT-NeoX (Pythia) is fused for full-rank training here", args)
    why = why or _neox_refusal(model) or native_attention_refusal(model.config.hidden_size // model.config.num_attention_heads, args)
    why = why or device_refusal(model)
    return (False, why) if why else (True, "ok")


class _Layer(LayerViews):
    __slots__ = ("W_qkv", "W_o", "W_h", "W_4", "A_qkv", "B_qkv", "b_qkv", "A_o", "B_o", "b_o", "A_h", "B_h", "b_h", "A_4", "B_4", "b_4",
                 "w1", "c1", "w2", "c2", "gA_qkv", "gB_qkv", "gb_qkv", "gA_o", "gB_o", "gb_o", "gA_h", "gB_h", "gb_h", "gA_4", "gB_4",
                 "gb_4", "gw1", "gc1", "gw2", "gc2", "key_qkv", "key_o", "key_h", "key_4", "mods", "merge", "gW_qkv", "gW_o", "gW_h",
                 "gW_4")


class FusedPythiaStepper(FusedStepperBase):
    """``model`` is a ``ReLoRaModel`` around a GPT-NeoX (ReLoRA: frozen weights, trainable LoRA factors) or a bare
    ``GPTNeoXForCausalLM`` (full-rank training: the projection weights are trainable and live in the flat store; every projection
    is the ReLoRA one without its low-rank branch).  ``quantize="mxfp8"``: the model's frozen weights are MXFP8-packed
    (``--quantize 8bit``) and stay so; the projections then run on the block-scaled GEMM (csrc/gemm_mx.cu)."""

    def __init__(self, model, info: DistInfo, *, lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, clip_grad_norm: float = 1.0, grad_accumulation: int = 1, zero: bool = False,
                 transport: str = "nccl", native=None, cuda_graphs: bool = True, ce_chunk: int = 4096,
                 overlap_wgrad: bool = True, attention: str = "auto", deterministic: bool = False, quantize: Optional[str] = None,
                 fp8: bool = False, activation_checkpointing: bool = False):
        if quantize is not None and canonical_format(quantize) != "mxfp8":
            raise RuntimeError(f"quantize={quantize!r}: only mxfp8 frozen weights run on the fused executor")
        if quantize is not None and fp8:
            raise RuntimeError("--frozen_dtype fp8 cannot be combined with --quantize: the frozen weights are already MXFP8")
        if fp8:
            raise RuntimeError("fp8 frozen weights are not supported for Pythia")
        super().__init__(model, info, supports_quantized if quantize is not None else supports, supports_full_rank,
                         grad_accumulation=grad_accumulation,
                         clip_grad_norm=clip_grad_norm, cuda_graphs=cuda_graphs, ce_chunk=ce_chunk, overlap_wgrad=overlap_wgrad,
                         attention=attention, deterministic=deterministic, activation_checkpointing=activation_checkpointing)
        neox = self.inner.gpt_neox
        layers = neox.layers
        self.parallel = bool(layers[0].use_parallel_residual)
        self.tanh = layers[0].mlp.act.approximate == "tanh"
        self.eps = [(l.input_layernorm.eps, l.post_attention_layernorm.eps) for l in layers]
        self.eps_f = neox.final_layer_norm.eps
        at0 = layers[0].attention
        self.rot = at0.rotary_ndims
        self.rotary = at0.rotary_emb
        self.mx = quantize is not None
        self.Wmx: List[List[mx.MxWeight]] = []  # per layer: the packed query_key_value, dense, dense_h_to_4h, dense_4h_to_h

        # ---------------------------------------------------------------- flat trainable store
        params: List[torch.nn.Parameter] = []
        for layer in layers:
            at, mlp = layer.attention, layer.mlp
            for m in (at.query_key_value, at.dense, mlp.dense_h_to_4h, mlp.dense_4h_to_h):
                params += [m.weight, m.bias] if self.full else [m.lora_A.weight, m.lora_B.weight, m.bias]
            for ln in (layer.input_layernorm, layer.post_attention_layernorm):
                params += [ln.weight, ln.bias]
        params += [neox.embed_in.weight, neox.final_layer_norm.weight, neox.final_layer_norm.bias, self.inner.embed_out.weight]
        self._build_store(params, transport)
        pv = self._stacked_view

        self.layers: List[_Layer] = []
        for layer in layers:
            at, mlp = layer.attention, layer.mlp
            S = _Layer()
            for tag, m in (("qkv", at.query_key_value), ("o", at.dense), ("h", mlp.dense_h_to_4h), ("4", mlp.dense_4h_to_h)):
                if self.full:
                    # trainable weight, [out, in] in the flat store; query_key_value's rows are in the head-interleaved order
                    # of dqkv, so its gradient needs no permutation
                    W, gW = pv(m.weight)
                    b, gb = pv(m.bias)
                    for k, v in (("W_", W), ("gW_", gW), ("b_", b), ("gb_", gb)):
                        setattr(S, k + tag, v)
                    # sanity: the store views must alias the module parameters
                    assert W.data_ptr() == m.weight.data_ptr() and W.shape == m.weight.shape
                    assert b.data_ptr() == m.bias.data_ptr()
                    continue
                # frozen weight: [out, in] contiguous as the module keeps it, or its packed bytes (``m.weight`` would be a transient
                # dequantised copy)
                setattr(S, "W_" + tag, m.qweight if self.mx else m.weight.data)
                A, gA = pv(m.lora_A.weight)
                B, gB = pv(m.lora_B.weight)
                b, gb = pv(m.bias)
                for k, v in (("A_", A), ("gA_", gA), ("B_", B), ("gB_", gB), ("b_", b), ("gb_", gb)):
                    setattr(S, k + tag, v)
                setattr(S, "key_" + tag, m.module_index + 1)  # LoRA-dropout mask stream of the module path
                assert A.data_ptr() == m.lora_A.weight.data_ptr() and b.data_ptr() == m.bias.data_ptr()
            S.w1, S.gw1 = pv(layer.input_layernorm.weight)
            S.c1, S.gc1 = pv(layer.input_layernorm.bias)
            S.w2, S.gw2 = pv(layer.post_attention_layernorm.weight)
            S.c2, S.gc2 = pv(layer.post_attention_layernorm.bias)
            S.mods = (at.query_key_value, at.dense, mlp.dense_h_to_4h, mlp.dense_4h_to_h)
            if self.mx:  # one packed weight per module: its (B, A, first row) block of the merge's fp32 delta s·B·A
                if not all(isinstance(m.qweight, mx.MxWeight) for m in S.mods):
                    raise RuntimeError("quantized frozen weights must be in the tensor-core layout (packed on the GPU)")
                self.Wmx.append([m.qweight for m in S.mods])
                S.merge = [[(m.lora_B.weight.data, m.lora_A.weight.data, 0)] for m in S.mods]
            elif not self.full:  # (B, A, W) blocks of the merge GEMM  W += s·B·A
                S.merge = [(m.lora_B.weight.data, m.lora_A.weight.data, m.weight.data) for m in S.mods]
            self.layers.append(S)
        self.W_emb, self.gW_emb = pv(neox.embed_in.weight)
        self.pad_idx = -1
        self.w_norm, self.gw_norm = pv(neox.final_layer_norm.weight)
        self.c_norm, self.gc_norm = pv(neox.final_layer_norm.bias)
        self.W_head, self.gW_head = pv(self.inner.embed_out.weight)

        # ---------------------------------------------------------------- optimizer / comm
        self._init_optimizer(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, zero=zero, native=native)
        self.dx_split_k = self.dx_split_k or 4096
        # --deterministic (full-rank training only; ReLoRA ignores it): the weight-gradient GEMMs run without split-K, so one CTA owns
        # an output tile for the whole token reduction.  The 1-D gradients (LayerNorm γ / β and the projection biases) stay column
        # sums whose block partials meet in fp32 atomics.
        self.wgrad_split_k = 1 if (self.full and self.deterministic) else 0

    # ------------------------------------------------------------------ buffers
    def _alloc_layers(self, B: int, T: int):
        dev, h, f, r, M = self.device, self.h, self.f, self.r, self.M_
        L = self.n_slots
        e = lambda *s: torch.empty(*s, dtype=BF, device=dev)  # noqa: E731
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
        # saved for the backward, one slot per layer or two under activation checkpointing ([0] only in evaluation)
        self.mean1, self.rstd1 = f32(L, M), f32(L, M)
        self.xd1, self.xd2 = e(L, M, h), e(L, M, h)  # LoRA inputs of query_key_value / dense_h_to_4h (the norms' outputs when p = 0)
        self.qkv = e(L, M, 3 * h)                    # post-rotary, head-interleaved
        self.xd_o = e(L, M, h)                       # attention output (dropout copy when p > 0): LoRA input of dense
        self.z = e(L, M, f)                          # pre-GELU
        self.xd_4 = e(L, M, f)                       # GELU output (dropout copy when p > 0): LoRA input of dense_4h_to_h
        if self.full:  # no low-rank branch: no u / du buffers, and the input gradient needs no separate base product
            self.u_qkv = self.u_o = self.u_h = self.u_4 = [None] * L
        else:
            self.u_qkv, self.u_o, self.u_h, self.u_4 = e(L, M, r), e(L, M, r), e(L, M, r), e(L, M, r)
        if not self.parallel:
            self.x1 = e(L, M, h)
            self.mean2, self.rstd2 = f32(L, M), f32(L, M)
        self._slotted = [self.mean1, self.rstd1, self.xd1, self.xd2, self.qkv, self.xd_o, self.z, self.xd_4]
        self._slotted += [] if self.full else [self.u_qkv, self.u_o, self.u_h, self.u_4]
        self._slotted += [] if self.parallel else [self.x1, self.mean2, self.rstd2]
        # transients
        self.xn1, self.xn2, self.attn_t, self.x1_t = e(M, h), e(M, h), e(M, h), e(M, h)
        self.a = e(M, f)
        self.mean_f, self.rstd_f = f32(M), f32(M)
        self.xf, self.dxf = e(M, h), e(M, h)
        self.dx_a, self.dx_b, self.dxn1, self.dxn2, self.dattn = e(M, h), e(M, h), e(M, h), e(M, h), e(M, h)
        self.dqkv = e(M, 3 * h)
        self.da, self.dz = e(M, f), e(M, f)
        if self.full:
            self.tmp_h = self.tmp_f = None
        else:
            self.tmp_h, self.tmp_f = e(M, h), e(M, f)
            self.du_bufs = {"4": e(M, r), "h": e(M, r), "o": e(M, r), "qkv": e(M, r)}
        if self.mx:
            # E4M3 rows + block scales of every GEMM input, [M, width] per width: the norms' and the attention outputs (h), the
            # GELU output (f) and the output gradients (h, f, 3h), each quantised right before the GEMM that reads it.  Zeros: the
            # scale bytes of the rows past M, which no call writes, are those mx_quantize_rows gives zero rows.
            u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8, device=dev)  # noqa: E731
            self.xq = {w: (u8(M, w), u8(self.C.mx_sf_bytes(M, w))) for w in (h, f, 3 * h)}
        # rotary tables of the module (linear / dynamic-NTK scaling, T beyond max_position_embeddings), fp32 [T, rot]
        if self.rot > 0:
            cos, sin = self.rotary(self.x_in, seq_len=T)
            self.cos = cos[0, 0, :T].float().contiguous()
            self.sin = sin[0, 0, :T].float().contiguous()

    # ------------------------------------------------------------------ forward
    def _attention(self, qkv: torch.Tensor, train: bool, al: int, out: torch.Tensor, keep: Optional[int] = None):
        """Attention of one layer into ``out``; ``al`` indexes the wgmma kernels' saved log-sum-exp, ``keep`` is ``_sdpa``'s."""
        B, T, nh, hd = self.B_, self.T_, self.nh, self.hd
        if self.native_attn:
            self.C.attention_fwd(qkv, out, self.lse[al], B, T, nh, hd, 1.0 / math.sqrt(hd), interleaved=True)
            return out
        v5 = qkv.view(B, T, nh, 3, hd)
        q, k, v = (v5[:, :, :, i].transpose(1, 2) for i in range(3))
        out.view(B, T, nh, hd).copy_(self._sdpa(q, k, v, train, keep).transpose(1, 2))
        return out

    def _norms(self, x, S, l, sl, train, p, both: bool, second_of=None):
        """LN1(x) (and LN2(x) when ``both``) or, with ``second_of``, LN2 of that input alone; returns the normed outputs and the LoRA
        inputs (dropout copies in training with p > 0)."""
        C, seed = self.C, self.seed
        keep = train and self.p == 0  # the normed output itself is the saved LoRA input
        outs = []
        specs = [(S.w2, S.c2, self.xd2, self.xn2, S.key_h)] if second_of is not None else \
            [(S.w1, S.c1, self.xd1, self.xn1, S.key_qkv)] + ([(S.w2, S.c2, self.xd2, self.xn2, S.key_h)] if both else [])
        for w, c, xd_buf, xn_t, key in specs:
            xn = xd_buf[sl] if keep else xn_t
            xd = xd_buf[sl] if (train and p > 0) else None
            outs.append((w, c, xn, xd, key))
        if second_of is not None:
            mean, rstd, eps = self.mean2[sl], self.rstd2[sl], self.eps[l][1]
        else:
            mean, rstd, eps = self.mean1[sl], self.rstd1[sl], self.eps[l][0]
        (w1, c1, y1, d1, k1) = outs[0]
        kw = {}
        if len(outs) == 2:
            (w2, c2, y2, d2, k2) = outs[1]
            kw = dict(w2=w2, b2=c2, y2=y2, xd2=d2)
        else:
            k2, d2 = 0, None
        if d1 is not None or d2 is not None:
            kw.update(xd=d1, seed=seed, keys=[k1, k2], p=p)
        C.layernorm_fwd(x, w1, c1, y1, mean, rstd, eps, **kw)
        return [(o[2], o[3] if o[3] is not None else o[2]) for o in outs]

    def _forward(self, train: bool):
        self.C.embedding_fwd(self.ids.view(-1), self.W_emb, self.x_in[0])
        self._attn_saved.clear()
        for l, S, sl, x, x_next in self._layer_slots(train):
            self._layer_fwd(l, S, sl, x, x_next, train)
        self.C.layernorm_fwd(x_next, self.w_norm, self.c_norm, self.xf, self.mean_f, self.rstd_f, self.eps_f)
        return x_next

    def _layer_fwd(self, l, S, sl, x, x_next, train, recompute=False):
        """One GPT-NeoX layer (see the base class).  A recompute reads the wgmma attention's saved output (SDPA runs again and keeps
        its graph) and forms only the LoRA product u of the projections that write no saved activation: dense_4h_to_h and, under
        parallel residual, dense, whose sum x1 only feeds x_next."""
        C, h, f = self.C, self.h, self.f
        p = self.p if train else 0.0
        seed = self.seed
        qkv = self.qkv[sl]
        normed = self._norms(x, S, l, sl, train, p, both=self.parallel)
        xn1, xd1 = normed[0]
        # ---- attention: qkv = [xn1 | u]·[W | B]ᵀ + b, rotary in place, attention on the interleaved layout
        self._lora_group_fwd(xn1, xd1, S.A_qkv, S.B_qkv, S.W_qkv, self.u_qkv[sl], qkv, G=1, K=h, Ng=3 * h, bias=S.b_qkv)
        if self.rot > 0:
            C.neox_rope(qkv, self.T_, self.nh, self.hd, self.rot, self.cos, self.sin, 0, False)
        al = l if train else 0
        out = self.attn_o[al] if self.native_attn else (self.xd_o[sl] if train and self.p == 0 else self.attn_t)
        attn = out if recompute and self.native_attn else self._attention(qkv, train, al, out, self._sdpa_keep(l, train, recompute))
        if p > 0:
            xd_o = self.xd_o[sl]
            C.dropout_expand(attn, xd_o, seed, [S.key_o], p)
        else:
            xd_o = attn
            if train and attn.data_ptr() != self.xd_o[sl].data_ptr():
                self.xd_o[sl].copy_(attn)
        x1 = self.x1[sl] if (train and not self.parallel) else self.x1_t
        self._lora_group_fwd(attn, xd_o, S.A_o, S.B_o, S.W_o, self.u_o[sl], x1, G=1, K=h, Ng=h, residual=x, bias=S.b_o,
                             u_only=recompute and self.parallel)
        # ---- MLP: z = [xn2 | u]·[W | B]ᵀ + b, GELU (+ dropout copy), x_next = [a | u]·[W | B]ᵀ + b + x1
        if self.parallel:
            xn2, xd2 = normed[1]
        else:
            xn2, xd2 = self._norms(x1, S, l, sl, train, p, both=False, second_of=x1)[0]
        z = self.z[sl]
        self._lora_group_fwd(xn2, xd2, S.A_h, S.B_h, S.W_h, self.u_h[sl], z, G=1, K=h, Ng=f, bias=S.b_h)
        a = self.xd_4[sl] if (train and self.p == 0) else self.a
        if p > 0:
            xd_4 = self.xd_4[sl]
            C.gelu_fwd(z, a, self.tanh, xd=xd_4, seed=seed, key=S.key_4, p=p)
        else:
            C.gelu_fwd(z, a, self.tanh)
            xd_4 = a
        self._lora_group_fwd(a, xd_4, S.A_4, S.B_4, S.W_4, self.u_4[sl], x_next, G=1, K=f, Ng=h, residual=x1, bias=S.b_4,
                             u_only=recompute)

    # ------------------------------------------------------------------ backward
    def _backward(self):
        C, h, f = self.C, self.h, self.f
        B, T, nh, hd = self.B_, self.T_, self.nh, self.hd
        dx, dx_other = self.dx_a, self.dx_b
        C.layernorm_bwd(self.dxf, self.x_in[self.L], self.w_norm, self.mean_f, self.rstd_f, dx, self.gw_norm, self.gc_norm)
        for l in range(self.L - 1, -1, -1):
            S, sl = self.layers[l], self._slot(l)
            # activation checkpointing: layer l into slot l % 2 (see _recompute).  Pending on the side stream are layer l + 1's
            # query_key_value weight gradients alone (its _join("o") covered the three groups it forked before), which read slot
            # (l + 1) % 2; layer l + 2's, the slot's previous readers, were all joined by layer l + 1's _join("qkv").
            self._recompute(l)
            # ---- MLP: x_next = a·W_4ᵀ + u_4·B_4ᵀ + b_4 + x1   (output gradient dx)
            self._lora_group_bwd(dx, S.B_4, S.W_4, S.A_4, S.gA_4, S.gB_4, self.xd_4[sl], self.u_4[sl], [S.key_4],
                                 G=1, K=f, Ng=h, base_out=self.tmp_f, out=self.da, tag="4", gW=S.gW_4)
            self._join("h")  # the previous layer's dense_h_to_4h weight gradients read dz / du
            C.gelu_bwd(self.da, self.z[sl], self.dz, self.tanh, dbias=S.gb_h)
            self._lora_group_bwd(self.dz, S.B_h, S.W_h, S.A_h, S.gA_h, S.gB_h, self.xd2[sl], self.u_h[sl], [S.key_h],
                                 G=1, K=h, Ng=f, base_out=self.tmp_h, out=self.dxn2, tag="h", gW=S.gW_h)
            if self.parallel:
                d_attn_out = dx  # dense's output gradient is the block's
            else:
                # x_next = x1 + mlp(LN2 x1) + b_4:  dx1 = dx + LN2ᵀ(dxn2); Σ dx is the bias gradient of dense_4h_to_h
                C.layernorm_bwd(self.dxn2, self.x1[sl], S.w2, self.mean2[sl], self.rstd2[sl], dx_other, S.gw2, S.gc2, dres=dx,
                                dres_sum=S.gb_4)
                dx, dx_other = dx_other, dx
                d_attn_out = dx
            # ---- attention: x1 = attn·W_oᵀ + u_o·B_oᵀ + b_o + x
            self._lora_group_bwd(d_attn_out, S.B_o, S.W_o, S.A_o, S.gA_o, S.gB_o, self.xd_o[sl], self.u_o[sl], [S.key_o],
                                 G=1, K=h, Ng=h, base_out=self.tmp_h, out=self.dattn, tag="o", gW=S.gW_o)
            if self.native_attn:
                self._join("qkv")  # the previous layer's query_key_value weight gradients read dqkv / du
                C.attention_bwd(self.qkv[sl], self.attn_o[l], self.dattn, self.lse[l], self.delta, self.dqkv, B, T, nh, hd,
                                1.0 / math.sqrt(hd), interleaved=True)
            else:
                dq, dk, dv = self._sdpa_bwd(l)
                self._join("qkv")
                d5 = self.dqkv.view(B, T, nh, 3, hd)
                for i, d in enumerate((dq, dk, dv)):
                    d5[:, :, :, i].copy_(d.transpose(1, 2))
            if self.rot > 0:
                C.neox_rope(self.dqkv, T, nh, hd, self.rot, self.cos, self.sin, 0, True)  # back through the rotation of q, k
            C.colsum(self.dqkv, S.gb_qkv)
            self._lora_group_bwd(self.dqkv, S.B_qkv, S.W_qkv, S.A_qkv, S.gA_qkv, S.gB_qkv, self.xd1[sl], self.u_qkv[sl], [S.key_qkv],
                                 G=1, K=h, Ng=3 * h, base_out=self.tmp_h, out=self.dxn1, tag="qkv", gW=S.gW_qkv)
            self._join("o")  # this layer's dense / dense_4h_to_h weight gradients read the buffer written next
            if self.parallel:
                # dx = dx_next + LN1ᵀ(dxn1) + LN2ᵀ(dxn2); Σ dx_next is the bias gradient of both dense and dense_4h_to_h
                C.layernorm_bwd(self.dxn1, self.x_in[l], S.w1, self.mean1[sl], self.rstd1[sl], dx_other, S.gw1, S.gc1, dres=dx,
                                dy2=self.dxn2, w2=S.w2, dw2=S.gw2, db2=S.gc2, dres_sum=S.gb_o, dres_sum2=S.gb_4)
            else:
                C.layernorm_bwd(self.dxn1, self.x_in[l], S.w1, self.mean1[sl], self.rstd1[sl], dx_other, S.gw1, S.gc1, dres=dx,
                                dres_sum=S.gb_o)
            dx, dx_other = dx_other, dx
        self._embedding_bwd_and_join(dx, ("4", "h", "o", "qkv"))
