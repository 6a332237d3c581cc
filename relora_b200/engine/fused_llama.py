"""Whole-model fused executor for Llama + ReLoRA on H100.

The reference executes one ``ReLoRaLinear`` as ~8 eager kernels (``relora.py:319-322``) and a decoder
layer as ~100 (``modeling_llama.py:243-308``), re-reading every activation several times, and is
launch/CPU-bound at the 250M scale.  This executor instead

* keeps the frozen weights of a layer *stacked* (``Wqkv [h + 2·kv, h]`` with kv = nkv·head_dim, i.e. ``[3h, h]`` without
  grouped-query attention; ``Wgu [2f,h]``) and the LoRA factors stacked alongside (``A_qkv [3r,h]``, ``B_qkv [h + 2·kv, r]`` …) —
  the ``nn.Module`` parameters are views into these buffers, so checkpoints keep the reference layout.  Under grouped-query
  attention the q group and the equal-width k | v groups of the stacked projections run as two launches into column windows;
* runs every projection as ONE wgmma GEMM launch with the low-rank up-projection folded into the K loop
  (``y = [x | u]·[W | B]ᵀ``, residual add in the epilogue), the three / two down-projections of a stacked group
  as one grouped launch, and all backward GEMMs (``dx``, ``du``, stacked ``dA`` / ``dB`` with split-K) on the same
  kernel reading operands MN-major in place — no transposed copies, no autograd graph;
* fuses RMSNorm with the LoRA-dropout expansion, computes LM-head + cross-entropy chunk-wise without ever
  materialising ``[tokens, V]`` logits, accumulates all gradients in one flat fp32 buffer;
* captures forward+backward of a micro-batch in a CUDA graph (dropout seeds live on the device and advance
  inside the graph), so a micro-step costs one graph launch on the host.

Full-rank training (a bare ``LlamaForCausalLM``, ``--engine fused``) runs the same layer loop without the low-rank branch: the
projection weights are trainable, live in the flat store as stacked views, and their fp32 gradients ``gW += dyᵀ·x`` run on the
side stream where ``dA`` / ``dB`` run under ReLoRA.

Math per layer (training, dropout p, scale s): see ``ops/reference.py`` — numerics tests compare this executor
with the module-by-module PyTorch path on identical weights and masks.
"""
from __future__ import annotations

import argparse
import math
import os
from typing import Dict, List, Optional, Tuple

import torch

from ..models.llama import LlamaForCausalLM, num_kv_heads
from ..ops import fused, mx, native
from ..ops.quant import canonical_format
from ..parallel.dist import DistInfo
from ..parallel.flat import _ALIGN as _STORE_ALIGN
from ..relora import ReLoRaLinear, ReLoRaModel
from .fused_common import (FusedStepperBase, LayerViews, checkpointing_refusal, device_refusal, full_rank_refusal,
                           native_attention_refusal, relora_refusal)

BF = torch.bfloat16


def supports(model, args=None) -> Tuple[bool, str]:
    why = relora_refusal(model, LlamaForCausalLM, "only Llama is fused") or checkpointing_refusal(args)
    if why:
        return False, why
    return _relora_shapes(model, args)


def supports_quantized(model, args=None) -> Tuple[bool, str]:
    """Whether the executor can train ``model`` with MXFP8-packed frozen weights (``--engine fused --quantize 8bit``), and if
    not, why.  ``--engine auto`` does not ask: it keeps quantised models on the module path."""
    if not isinstance(model, ReLoRaModel):
        return False, "quantized frozen weights need a ReLoRA model; full-rank training has no frozen weights"
    if not isinstance(model.wrapped_model, LlamaForCausalLM):
        return False, "quantized frozen weights are fused for Llama only; other models use --engine module"
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
    if any(isinstance(m, ReLoRaLinear) and m.bias is not None for m in model.wrapped_model.modules()):
        return False, "biased projections use the module path"
    f = model.wrapped_model.config.intermediate_size
    if f % 8:
        # the module path keeps such weights in ops/quant.py's 1 x 32-block layout; repacking them into 32 x 32 tiles would round
        # the frozen weights a second time
        return False, f"quantized frozen weights need an intermediate size that is a multiple of 8 (got {f}) for the tensor-core layout"
    return _relora_shapes(model, args)


def _relora_shapes(model, args) -> Tuple[bool, str]:
    inner = model.wrapped_model
    cfg = inner.config
    h, f, nh = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads
    nkv = num_kv_heads(cfg)
    r = model.r
    hd = h // nh
    if nkv != nh:
        if nkv * hd % 128:
            return False, f"grouped-query attention needs num_key_value_heads x head_dim ({nkv} x {hd}) to be a multiple of 128"
        if getattr(args, "frozen_dtype", None) in ("fp8", "fp8_full"):
            return False, "--frozen_dtype fp8 with grouped-query attention uses the module path (the fp8 weight copies are [3h, h])"
    if h % 128 or r % 128:
        # the intermediate size may be anything (llama_1b: 5461): its buffers are zero-padded to a multiple of 128
        return False, f"hidden ({h}) and rank ({r}) must be multiples of 128 for stacked groups"
    if hd % 8 or hd % 4:
        return False, "head_dim must be a multiple of 8"
    # --attention native is not checked here but in the constructor: declining would send such a model to the module path
    why = device_refusal(inner)
    if why:
        return False, why
    for m in inner.modules():
        if isinstance(m, ReLoRaLinear) and m.bias is not None:
            return False, "biased projections use the module path"
    return True, "ok"


def supports_full_rank(model, args=None) -> Tuple[bool, str]:
    """Whether the executor can train ``model`` (an unwrapped Llama) full-rank, and if not, why."""
    why = full_rank_refusal(model, LlamaForCausalLM, "only Llama is fused for full-rank training", args)
    if why:
        return False, why
    cfg = model.config
    h, nh = cfg.hidden_size, cfg.num_attention_heads
    hd = h // nh
    kv = num_kv_heads(cfg) * hd
    # every GEMM operand is read through a TMA tensor map, whose row pitch must be a multiple of 16 bytes (gemm_wgmma.cu:
    # make_map_2d): x / dx [tokens, hidden], W and dW [*, hidden], and the packed q | k | v row of h + 2·kv
    if h % 8 or (h + 2 * kv) % 8:
        return False, f"hidden ({h}) and hidden + 2 x num_key_value_heads x head_dim ({h + 2 * kv}) must be multiples of 8 for the GEMM's 16-byte row pitch"
    # the stacked Wqkv view needs q / k / v adjacent in the flat store, whose segments start on 128-element boundaries
    if (h * h) % _STORE_ALIGN or (kv * h) % _STORE_ALIGN:
        return False, f"hidden x hidden ({h * h}) and kv width x hidden ({kv * h}) must be multiples of {_STORE_ALIGN} for the stacked q | k | v weights"
    if h > 8192:
        return False, f"hidden ({h}) is above the RMSNorm kernels' 8192"
    if hd % 8:
        return False, f"head_dim ({hd}) must be a multiple of 8 for the attention and RoPE kernels"
    why = native_attention_refusal(hd, args)
    if why:
        return False, why
    for m in model.modules():
        if isinstance(m, torch.nn.Linear) and m.bias is not None:
            return False, "biased projections use the module path"
    why = device_refusal(model)
    return (False, why) if why else (True, "ok")


class _Layer(LayerViews):
    __slots__ = ("Wqkv", "Wo", "Wgu", "Wd", "A_qkv", "B_qkv", "A_o", "B_o", "A_gu", "B_gu", "A_d", "B_d", "w1", "w2",
                 "gA_qkv", "gB_qkv", "gA_o", "gB_o", "gA_gu", "gB_gu", "gA_d", "gB_d", "gw1", "gw2", "keys_qkv", "key_o",
                 "keys_gu", "key_d", "mods", "merge", "gWqkv", "gWo", "gWgu", "gWd")


class FusedLlamaStepper(FusedStepperBase):
    """``model`` is a ``ReLoRaModel`` around a Llama (ReLoRA: frozen stacked weights, trainable LoRA factors) or a bare
    ``LlamaForCausalLM`` (full-rank training: the projection weights are trainable and live in the flat store; every projection
    is the ReLoRA one without its low-rank branch)."""

    def __init__(self, model, info: DistInfo, *, lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, clip_grad_norm: float = 1.0, grad_accumulation: int = 1, zero: bool = False,
                 transport: str = "nccl", native=None, cuda_graphs: bool = True, ce_chunk: int = 4096,
                 overlap_wgrad: bool = True, attention: str = "auto", fp8: bool = False, fp8_backward: bool = False,
                 deterministic: bool = False, quantize: Optional[str] = None, activation_checkpointing: bool = False):
        """``quantize="mxfp8"``: the model's frozen weights are MXFP8-packed (``--quantize 8bit``) and stay so; the stacks below
        are then packed too and the projections run on the block-scaled GEMM (csrc/gemm_mx.cu).  ``activation_checkpointing``:
        see ``FusedStepperBase``; the fp8 path is refused with it (``fused_common.checkpointing_refusal``)."""
        if quantize is not None and canonical_format(quantize) != "mxfp8":
            raise RuntimeError(f"quantize={quantize!r}: only mxfp8 frozen weights run on the fused executor")
        if quantize is not None and (fp8 or fp8_backward):
            raise RuntimeError("--frozen_dtype fp8 cannot be combined with --quantize: the frozen weights are already MXFP8")
        super().__init__(model, info, supports_quantized if quantize is not None else supports, supports_full_rank,
                         grad_accumulation=grad_accumulation,
                         clip_grad_norm=clip_grad_norm, cuda_graphs=cuda_graphs, ce_chunk=ce_chunk, overlap_wgrad=overlap_wgrad,
                         attention=attention, deterministic=deterministic, activation_checkpointing=activation_checkpointing)
        if self.full and fp8:
            raise RuntimeError("--frozen_dtype fp8 has no frozen weights to act on in full-rank training")
        if fp8 and num_kv_heads(model.wrapped_model.config) != model.wrapped_model.config.num_attention_heads:
            raise RuntimeError("--frozen_dtype fp8 with grouped-query attention uses the module path (the fp8 weight copies are [3h, h])")
        cfg = self.inner.config
        self.nkv = num_kv_heads(cfg)
        self.kv = self.nkv * self.hd  # width of the k and v projections (h without grouped-query attention)
        self.qkv_w = self.h + 2 * self.kv  # packed [q | k | v] row
        self.fp = (self.f + 127) // 128 * 128  # padded intermediate size (zero rows / columns keep every GEMM extent a multiple of the 128-wide tile)
        self.eps = cfg.rms_norm_eps

        # ---------------------------------------------------------------- stacked frozen weights (ReLoRA)
        dev = self.device
        h, f, fp, r, L = self.h, self.f, self.fp, self.r, self.L
        kv = self.kv
        layers = self.inner.model.layers
        self.Wqkv = self.Wo = self.Wgu = self.Wd = None  # full rank: the trainable weights are stacked views into the flat store
        self.mx = quantize is not None
        self.Wmx: List[List[mx.MxWeight]] = []  # per layer: the packed qkv, o, gate|up and down stacks
        if self.mx:
            self._pack_stacks(layers)
        elif not self.full:
            self.Wqkv = torch.empty(L, h + 2 * kv, h, dtype=BF, device=dev)
            self.Wo = torch.empty(L, h, h, dtype=BF, device=dev)
            self.Wgu = torch.zeros(L, 2 * fp, h, dtype=BF, device=dev)
            self.Wd = torch.zeros(L, h, fp, dtype=BF, device=dev)
            with torch.no_grad():
                for l, layer in enumerate(layers):
                    at, mlp = layer.self_attn, layer.mlp
                    for m, r0, r1 in ((at.q_proj, 0, h), (at.k_proj, h, h + kv), (at.v_proj, h + kv, h + 2 * kv)):
                        self._rehome(m.weight, self.Wqkv[l, r0:r1])
                    self._rehome(at.o_proj.weight, self.Wo[l])
                    self._rehome(mlp.gate_proj.weight, self.Wgu[l, :f])
                    self._rehome(mlp.up_proj.weight, self.Wgu[l, fp:fp + f])
                    self._rehome(mlp.down_proj.weight, self.Wd[l][:, :f])

        # ---------------------------------------------------------------- flat trainable store (stack-friendly order)
        params: List[torch.nn.Parameter] = []
        for layer in layers:
            at, mlp = layer.self_attn, layer.mlp
            if self.full:
                params += [m.weight for m in (at.q_proj, at.k_proj, at.v_proj, at.o_proj, mlp.gate_proj, mlp.up_proj, mlp.down_proj)]
            else:
                params += [m.lora_A.weight for m in (at.q_proj, at.k_proj, at.v_proj)]
                params += [m.lora_B.weight for m in (at.q_proj, at.k_proj, at.v_proj)]
                params += [at.o_proj.lora_A.weight, at.o_proj.lora_B.weight]
                params += [mlp.gate_proj.lora_A.weight, mlp.up_proj.lora_A.weight]
                params += [mlp.gate_proj.lora_B.weight, mlp.up_proj.lora_B.weight]
                params += [mlp.down_proj.lora_A.weight, mlp.down_proj.lora_B.weight]
            params += [layer.input_layernorm.weight, layer.post_attention_layernorm.weight]
        params += [self.inner.model.embed_tokens.weight, self.inner.model.norm.weight, self.inner.lm_head.weight]
        padded: Dict[int, Tuple[int, int]] = {}
        if fp != f:
            for layer in layers:
                mlp = layer.mlp
                if self.full:  # zero rows of gate / up and zero columns of down: zero gradients, so AdamW leaves them zero
                    padded[id(mlp.gate_proj.weight)] = (fp, h)
                    padded[id(mlp.up_proj.weight)] = (fp, h)
                    padded[id(mlp.down_proj.weight)] = (h, fp)
                    continue
                padded[id(mlp.gate_proj.lora_B.weight)] = (fp, r)
                padded[id(mlp.up_proj.lora_B.weight)] = (fp, r)
                padded[id(mlp.down_proj.lora_A.weight)] = (r, fp)
        self._build_store(params, transport, padded)
        pv = self._stacked_view  # stacked view over `rows_mult` adjacent parameters (params and grads)

        self.layers: List[_Layer] = []
        for layer in layers:
            at, mlp = layer.self_attn, layer.mlp
            S = _Layer()
            l = len(self.layers)
            S.w1, S.gw1 = pv(layer.input_layernorm.weight)
            S.w2, S.gw2 = pv(layer.post_attention_layernorm.weight)
            if self.full:
                S.Wqkv, S.gWqkv = pv(at.q_proj.weight, rows=h + 2 * kv)
                S.Wo, S.gWo = pv(at.o_proj.weight)
                S.Wgu, S.gWgu = pv(mlp.gate_proj.weight, 2)
                S.Wd, S.gWd = pv(mlp.down_proj.weight)
                # sanity: the stacked views must alias the module parameters
                assert S.Wqkv[h:h + kv].data_ptr() == at.k_proj.weight.data_ptr()
                assert S.Wqkv[h + kv:].data_ptr() == at.v_proj.weight.data_ptr() and S.Wqkv.shape == (h + 2 * kv, h)
                assert S.Wgu[fp:].data_ptr() == mlp.up_proj.weight.data_ptr() and S.Wgu.shape == (2 * fp, h)
                assert S.Wd.data_ptr() == mlp.down_proj.weight.data_ptr() and S.Wd.shape == (h, fp)
                self.layers.append(S)
                continue
            if self.mx:
                S.Wqkv, S.Wo, S.Wgu, S.Wd = self.Wmx[l]
            else:
                S.Wqkv, S.Wo, S.Wgu, S.Wd = self.Wqkv[l], self.Wo[l], self.Wgu[l], self.Wd[l]
            S.A_qkv, S.gA_qkv = pv(at.q_proj.lora_A.weight, 3)
            S.B_qkv, S.gB_qkv = pv(at.q_proj.lora_B.weight, 3) if kv == h else pv(at.q_proj.lora_B.weight, rows=h + 2 * kv)
            S.A_o, S.gA_o = pv(at.o_proj.lora_A.weight)
            S.B_o, S.gB_o = pv(at.o_proj.lora_B.weight)
            S.A_gu, S.gA_gu = pv(mlp.gate_proj.lora_A.weight, 2)
            S.B_gu, S.gB_gu = pv(mlp.gate_proj.lora_B.weight, 2)
            S.A_d, S.gA_d = pv(mlp.down_proj.lora_A.weight)
            S.B_d, S.gB_d = pv(mlp.down_proj.lora_B.weight)
            S.keys_qkv = [m.module_index + 1 for m in (at.q_proj, at.k_proj, at.v_proj)]
            S.key_o = at.o_proj.module_index + 1
            S.keys_gu = [mlp.gate_proj.module_index + 1, mlp.up_proj.module_index + 1]
            S.key_d = mlp.down_proj.module_index + 1
            S.mods = (at.q_proj, at.k_proj, at.v_proj, at.o_proj, mlp.gate_proj, mlp.up_proj, mlp.down_proj)
            # sanity: the stacked views must alias the module parameters
            assert S.A_qkv[r:2 * r].data_ptr() == at.k_proj.lora_A.weight.data_ptr()
            assert S.B_qkv[h + kv:].data_ptr() == at.v_proj.lora_B.weight.data_ptr() and S.B_qkv.shape == (h + 2 * kv, r)
            assert S.B_gu[fp:].data_ptr() == mlp.up_proj.lora_B.weight.data_ptr()
            assert S.A_d.data_ptr() == mlp.down_proj.lora_A.weight.data_ptr() and S.A_d.shape == (r, fp)
            if self.mx:  # (B, A, first stack row) of each module of each packed stack: the merge's fp32 delta s·B·A
                kvB = [S.B_qkv[:h], S.B_qkv[h:h + kv], S.B_qkv[h + kv:]]
                S.merge = [[(kvB[i], S.A_qkv[i * r:(i + 1) * r], (0, h, h + kv)[i]) for i in range(3)], [(S.B_o, S.A_o, 0)],
                           [(S.B_gu[:fp], S.A_gu[:r], 0), (S.B_gu[fp:], S.A_gu[r:], fp)], [(S.B_d, S.A_d, 0)]]
            else:
                # (B, A, W) blocks of the merge GEMM  W += s·B·A  (padded blocks where the module views are strided)
                S.merge = [(m.lora_B.weight.data, m.lora_A.weight.data, m.weight.data) for m in S.mods[:4]]
                S.merge += [(S.B_gu[:fp], S.A_gu[:r], S.Wgu[:fp]), (S.B_gu[fp:], S.A_gu[r:], S.Wgu[fp:]), (S.B_d, S.A_d, S.Wd)]
            self.layers.append(S)
        emb = self.inner.model.embed_tokens
        self.W_emb, self.gW_emb = pv(emb.weight)
        self.pad_idx = emb.padding_idx if emb.padding_idx is not None else -1
        self.w_norm, self.gw_norm = pv(self.inner.model.norm.weight)
        self.W_head, self.gW_head = pv(self.inner.lm_head.weight)

        rot = layers[0].self_attn.rotary_emb
        self.cos = rot.cos_cached[0, 0].to(BF).contiguous()
        self.sin = rot.sin_cached[0, 0].to(BF).contiguous()

        # ---------------------------------------------------------------- optimizer / comm
        self._init_optimizer(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, zero=zero, native=native)
        # ---- fp8 frozen-weight path: E4M3 copies of the stacked weights + per-site activation scales (csrc/fp8.cu)
        self.fp8 = not self.full and (bool(fp8) or os.environ.get("RELORA_B200_FP8", "0") == "1")
        why = checkpointing_refusal(argparse.Namespace(activation_checkpointing=self.recompute,
                                                       frozen_dtype="fp8" if self.fp8 else None))
        if why:
            raise RuntimeError(why)
        if self.fp8:
            u8 = lambda *sh: torch.zeros(*sh, dtype=torch.uint8, device=dev)  # noqa: E731
            self.W8 = [u8(L, 3 * h, h), u8(L, h, h), u8(L, 2 * fp, h), u8(L, h, fp)]  # sites: qkv, o, gate/up, down
            f32 = lambda *sh: torch.zeros(*sh, dtype=torch.float32, device=dev)  # noqa: E731
            # scale bookkeeping, index [direction, layer, site]: direction 0 = forward activations (E4M3), 1 = output gradients
            # (E5M2) of the same four projection groups
            self._w_scale2, self._act_state2 = f32(2, L, 4), f32(2, L, 4, 2)
            self._inv_sx2, self._alpha_main2, self._alpha_inv2 = f32(2, L, 4), f32(2, L, 4), f32(2, L, 4)
            self.w_scale, self.act_state = self._w_scale2[0], self._act_state2[0]
            self.inv_sx, self.alpha_main, self.alpha_inv = self._inv_sx2[0], self._alpha_main2[0], self._alpha_inv2[0]
            self.w_inv_scale, self._amax_scratch = f32(L, 4), f32(1)
            self.fp8_bwd = bool(fp8_backward) or os.environ.get("RELORA_B200_FP8_BWD", "0") == "1"
            self._fp8_bwd_calibrated = False
            # E4M3 copies of the transposed weights: K-major operands of the input-gradient GEMMs dy·W
            self.W8T = [u8(L, h, 3 * h), u8(L, h, h), u8(L, h, 2 * fp), u8(L, fp, h)] if self.fp8_bwd else None
            self.fp8_margin = float(os.environ.get("RELORA_B200_FP8_MARGIN", "1.5"))
            self._fp8_calibrated = False
            self._quantize_weights()
        self._fp8_calibrating = False
        self.fused_dx = os.environ.get("RELORA_B200_FUSED_DX", "1") != "0"
        # stacked output width from which dx uses two kernels (frozen-path GEMM on 256-wide tiles + a mask-and-add pass) instead of
        # the one-kernel form; the thresholds (4096 bf16, 2048 with fp8 input-gradient GEMMs) have not been re-tuned on the H100.
        self.dx_split_k = self.dx_split_k or (2048 if self.fp8_bwd else 4096)
        # --deterministic: the stacked dA / dB weight-gradient GEMMs run without split-K (one CTA owns an output tile for the whole token
        # reduction: fixed summation order instead of fp32 atomics from several CTAs).  Remaining order-dependent reductions are the
        # [h]-sized norm-weight gradients (block partials combined with vector atomics).
        self.wgrad_split_k = 1 if self.deterministic else 0

    # ------------------------------------------------------------------ plumbing
    @staticmethod
    def _rehome(param: torch.nn.Parameter, dst: torch.Tensor):
        dst.copy_(param.data)
        param.data = dst

    # (module, first stack row) of the qkv, o, gate|up and down stacks of a layer
    def _stack_rows(self, layer):
        at, mlp, h, kv, fp = layer.self_attn, layer.mlp, self.h, self.kv, self.fp
        return [[(at.q_proj, 0), (at.k_proj, h), (at.v_proj, h + kv)], [(at.o_proj, 0)], [(mlp.gate_proj, 0), (mlp.up_proj, fp)],
                [(mlp.down_proj, 0)]]

    @torch.no_grad()
    def _pack_stacks(self, layers):
        """The packed stacks of every layer, built from the modules' packed bytes as they are, then each module's ``qweight``
        re-pointed at its rows of them, so the stacks are the only resident copy of the frozen weights."""
        for layer in layers:
            stacks = []
            for group in self._stack_rows(layer):
                st = mx.stack_weights([m.qweight for m, _ in group])  # every part starts on a 128-row boundary
                for m, r0 in group:
                    m.qweight = mx.stack_part(st, r0, m.out_features)
                    m.qweight.K = m.in_features  # the down projection of a padded intermediate size: K is the module's own
                stacks.append(st)
            self.Wmx.append(stacks)

    @torch.no_grad()
    def _quantize_weights(self):
        """(Re)build the E4M3 copies of the frozen weights and their per-tensor scales (at start-up and after every merge)."""
        stacks = (self.Wqkv, self.Wo, self.Wgu, self.Wd)
        for l in range(self.L):
            for s_i in range(4):
                self.C.fp8_quantize_weight(stacks[s_i][l], self.W8[s_i][l], self._amax_scratch, self.w_scale[l, s_i:s_i + 1],
                                           self.w_inv_scale[l, s_i:s_i + 1], self.W8T[s_i][l] if self.fp8_bwd else None)
        self._w_scale2[1].copy_(self._w_scale2[0])

    def _alloc_layers(self, B: int, T: int):
        dev, h, f, r, M = self.device, self.h, self.fp, self.r, self.M_  # f: padded intermediate size
        L = self.n_slots  # saved for the backward: one slot per layer, or two under activation checkpointing
        e = lambda *s: torch.empty(*s, dtype=BF, device=dev)  # noqa: E731
        self.x1 = e(L, M, h)
        self.rstd1 = torch.empty(L, M, dtype=torch.float32, device=dev)
        self.rstd2 = torch.empty(L, M, dtype=torch.float32, device=dev)
        self.rstd_f = torch.empty(M, dtype=torch.float32, device=dev)
        G3, G2 = (3, 2) if self.p > 0 else (1, 1)
        self.xd_qkv = e(L, M, G3 * h)
        self.xd_o = e(L, M, h)
        self.xd_gu = e(L, M, G2 * h)
        self.xd_d = e(L, M, f)
        self.qkv = e(L, M, self.qkv_w)
        self.gu = e(L, M, 2 * f)
        # transients
        self.xn = e(M, h)
        self.hmid = e(M, f)
        self.xf = e(M, h)
        self.dxf = e(M, h)
        self.dx_a, self.dx_b, self.dxn2 = e(M, h), e(M, h), e(M, h)
        self.dattn = e(M, h)
        self.dqkv = e(M, self.qkv_w)
        self.dgu = e(M, 2 * f)
        self.dhmid2 = e(M, f)
        if self.full:
            # no low-rank branch: the input gradient is one GEMM straight into its output, so there are no u / du buffers and
            # no separate base product (dxn, dhmid, parts)
            self.u_qkv = self.u_o = self.u_gu = self.u_d = [None] * L
            self.dxn = self.dhmid = None
        else:
            self.u_qkv = e(L, M, 3 * r)
            self.u_o = e(L, M, r)
            self.u_gu = e(L, M, 2 * r)
            self.u_d = e(L, M, r)
            self.dxn, self.dhmid = e(M, h), e(M, f)
            self.du_bufs = {"d": e(M, r), "gu": e(M, 2 * r), "o": e(M, r), "qkv": e(M, 3 * r)}
        self._slotted = [self.x1, self.rstd1, self.rstd2, self.xd_qkv, self.xd_o, self.xd_gu, self.xd_d, self.qkv, self.gu]
        if not self.full:
            self._slotted += [self.u_qkv, self.u_o, self.u_gu, self.u_d]
        if self.mx:  # E4M3 rows + block scales of every GEMM input: [M, width] per width
            widths = {h, f, self.qkv_w, 2 * f}
            # zeros: the scale bytes of the rows past M that no producer writes are those mx_quantize_rows gives zero rows
            self.xq = {w: (torch.empty(M, w, dtype=torch.uint8, device=dev),
                           torch.zeros(self.C.mx_sf_bytes(M, w), dtype=torch.uint8, device=dev)) for w in widths}
        if self.fp8:
            self.x8_h = torch.empty(M, h, dtype=torch.uint8, device=dev)
            self.x8_f = torch.empty(M, f, dtype=torch.uint8, device=dev)
            if self.fp8_bwd:
                self.dy8 = {w: torch.empty(M, w, dtype=torch.uint8, device=dev) for w in {h, 3 * h, 2 * f}}
        self.parts = None if self.full else e(M, max(3 * h, f))

    # ------------------------------------------------------------------ forward + backward of one micro-batch
    def _attention(self, qkv: torch.Tensor, train: bool, al: int = 0, keep: Optional[int] = None):
        """Attention of one layer; ``al`` indexes the wgmma kernels' saved output and log-sum-exp, ``keep`` is ``_sdpa``'s."""
        B, T, nh, hd = self.B_, self.T_, self.nh, self.hd
        if self.native_attn:
            # wgmma flash attention straight out of the packed projection buffer (csrc/attention.cu); the output and the
            # log-sum-exp of the layer are what the backward kernels need
            out = self.attn_o[al]
            if self.nkv == nh:
                self.C.attention_fwd(qkv, out, self.lse[al], B, T, nh, hd, 1.0 / math.sqrt(hd))
            else:
                self.C.attention_fwd(qkv, out, self.lse[al], B, T, nh, hd, 1.0 / math.sqrt(hd), nkv=self.nkv)
            return out
        if self.nkv == nh:
            v5 = qkv.view(B, T, 3, nh, hd)
            q, k, v = (v5[:, :, i].transpose(1, 2) for i in range(3))
            gqa = {}
        else:  # [q: nh | k: nkv | v: nkv] heads of the packed row
            v3 = qkv.view(B, T, nh + 2 * self.nkv, hd)
            q, k, v = (v3[:, :, a:b].transpose(1, 2) for a, b in ((0, nh), (nh, nh + self.nkv), (nh + self.nkv, nh + 2 * self.nkv)))
            gqa = {"enable_gqa": True}
        return self._sdpa(q, k, v, train, keep, **gqa).transpose(1, 2).reshape(self.M_, self.h)

    def _q8(self, l, s_i, K):
        """(q8, inv_scale, amax_cur) arguments that make a producer kernel also emit the E4M3 copy of its output; on packed
        stacks, the MX rows of its [M, K] output (see ``_mx``) for the norms and SwiGLU, none for the attention's dropout copy
        (site 1: the o projection quantises the attention output itself)."""
        if self.mx:
            return (self.xq[K][0], None, self.xq[K][1]) if s_i != 1 else (None, None, None)
        if not self.fp8:
            return (None, None, None)
        return (self.x8_h if K == self.h else self.x8_f, self.inv_sx[l, s_i:s_i + 1], self.act_state[l, s_i, 1:2])

    def _mx(self, K):
        """Keyword arguments that make a producer kernel also emit the MX rows of its [M, K] output (the next GEMM's input)."""
        return dict(q8=self.xq[K][0], q_amax=self.xq[K][1]) if self.mx else {}  # no q_inv_scale: the MX form

    def _forward(self, train: bool):
        if train and self.fp8 and not self._fp8_calibrating:
            self._fp8_prep()
        self.C.embedding_fwd(self.ids.view(-1), self.W_emb, self.x_in[0])
        self._attn_saved.clear()
        for l, S, sl, x, x_next in self._layer_slots(train):
            self._layer_fwd(l, S, sl, x, x_next, train)
        self.C.rmsnorm_fwd(x_next, self.w_norm, self.xf, self.rstd_f, self.eps, None, None, [], 0.0)
        return x_next

    def _layer_fwd(self, l, S, sl, x, x_next, train, recompute=False):
        """One decoder layer (see the base class).  A recompute reads the wgmma attention's saved output (SDPA runs again and keeps
        its graph) and forms only the down projection's LoRA product u_d, since x_next is saved."""
        C, M, h, f = self.C, self.M_, self.h, self.fp
        p = self.p if train else 0.0
        seed = self.seed
        x1 = self.x1[sl]
        qkv, gu = self.qkv[sl], self.gu[sl]
        # ---- attention block
        if p > 0:
            xd = self.xd_qkv[sl]
            C.rmsnorm_fwd(x, S.w1, self.xn, self.rstd1[sl], self.eps, xd, seed, S.keys_qkv, p, *self._q8(l, 0, h))
            xn = self.xn
        else:
            xn = self.xd_qkv[sl][:, :h] if self.p == 0 else self.xn  # p==0: the normed input is what dA needs
            xn = xn if xn.is_contiguous() else self.xn
            C.rmsnorm_fwd(x, S.w1, xn, self.rstd1[sl], self.eps, None, None, [], 0.0, **self._mx(h))
            xd = xn
        self._lora_group_fwd(xn, xd, S.A_qkv, S.B_qkv, S.Wqkv, self.u_qkv[sl], qkv, G=3, K=h, Ng=self.kv, site=(l, 0),
                             prequant=p > 0, Nq=h, mx_ready=True)
        C.rope_inplace(qkv, self.T_, self.nh + self.nkv, self.hd, self.hd, self.cos, self.sin, False, 0)
        if recompute and self.native_attn:
            attn = self.attn_o[l]
        else:
            attn = self._attention(qkv, train, l if train else 0, self._sdpa_keep(l, train, recompute))
        if p > 0:
            xd_o = self.xd_o[sl]
            C.dropout_expand(attn, xd_o, seed, [S.key_o], p, *self._q8(l, 1, h))
        else:
            xd_o = attn
            if train:
                self.xd_o[sl].copy_(attn)
        self._lora_group_fwd(attn, xd_o, S.A_o, S.B_o, S.Wo, self.u_o[sl], x1, G=1, K=h, Ng=h, residual=x, site=(l, 1), prequant=p > 0)
        # ---- MLP block
        if p > 0:
            xd = self.xd_gu[sl]
            C.rmsnorm_fwd(x1, S.w2, self.xn, self.rstd2[sl], self.eps, xd, seed, S.keys_gu, p, *self._q8(l, 2, h))
            xn = self.xn
        else:
            xn = self.xd_gu[sl] if self.p == 0 else self.xn
            C.rmsnorm_fwd(x1, S.w2, xn, self.rstd2[sl], self.eps, None, None, [], 0.0, **self._mx(h))
            xd = xn
        self._lora_group_fwd(xn, xd, S.A_gu, S.B_gu, S.Wgu, self.u_gu[sl], gu, G=2, K=h, Ng=f, site=(l, 2), prequant=p > 0,
                             mx_ready=True)
        if p > 0:
            xd_d = self.xd_d[sl]
            C.swiglu_fwd(gu, self.hmid, xd_d, seed, S.key_d, p, *self._q8(l, 3, f))  # activation, dropout copy (and E4M3 / MX copy)
        else:
            C.swiglu_fwd(gu, self.hmid, None, None, 0, 0.0, *self._q8(l, 3, f))
            xd_d = self.hmid
            if train:
                self.xd_d[sl].copy_(self.hmid)
        self._lora_group_fwd(self.hmid, xd_d, S.A_d, S.B_d, S.Wd, self.u_d[sl], x_next, G=1, K=f, Ng=h, residual=x1, site=(l, 3), prequant=True,
                             mx_ready=True, u_only=recompute)

    def _backward(self):
        C, g, M, h, f, r = self.C, fused.gemm, self.M_, self.h, self.fp, self.r
        B, T, nh, hd = self.B_, self.T_, self.nh, self.hd
        dx, dx_other = self.dx_a, self.dx_b
        ws, tk = fused.norm_workspace(self.device, h)
        C.rmsnorm_bwd(self.dxf, self.x_in[self.L], self.w_norm, self.rstd_f, None, dx, self.gw_norm, ws, tk)
        for l in range(self.L - 1, -1, -1):
            S, sl = self.layers[l], self._slot(l)
            # activation checkpointing: layer l into slot l % 2 (see _recompute).  Pending on the side stream are layer l + 1's
            # gate/up, o and qkv weight gradients (its down_proj ones were joined at the end of its backward), which read slot
            # (l + 1) % 2; layer l + 2's, the slot's previous readers, were all joined by layer l + 1's _join("qkv").
            self._recompute(l)
            # ---- MLP: x_next = hmid·Wdᵀ + u_d·B_dᵀ + x1
            self._lora_group_bwd(dx, S.B_d, S.Wd, S.A_d, S.gA_d, S.gB_d, self.xd_d[sl], self.u_d[sl], [S.key_d],
                                 G=1, K=f, Ng=h, base_out=self.dhmid, out=self.dhmid2, tag="d", site=(l, 3), gW=S.gWd)
            self._join("gu")  # the previous layer's gate/up weight gradients read dgu / du_gu
            C.swiglu_bwd(self.dhmid2, self.gu[sl], self.dgu)
            self._lora_group_bwd(self.dgu, S.B_gu, S.Wgu, S.A_gu, S.gA_gu, S.gB_gu, self.xd_gu[sl], self.u_gu[sl], S.keys_gu,
                                 G=2, K=h, Ng=f, base_out=self.dxn, out=self.dxn2, tag="gu", site=(l, 2), gW=S.gWgu)
            self._join("o")  # ... and its o_proj weight gradients read the buffer this norm backward writes
            C.rmsnorm_bwd(self.dxn2, self.x1[sl], S.w2, self.rstd2[sl], dx, dx_other, S.gw2, ws, tk)
            dx, dx_other = dx_other, dx  # dx = grad wrt x1
            # ---- attention: x1 = attn·Woᵀ + u_o·B_oᵀ + x
            self._lora_group_bwd(dx, S.B_o, S.Wo, S.A_o, S.gA_o, S.gB_o, self.xd_o[sl], self.u_o[sl], [S.key_o],
                                 G=1, K=h, Ng=h, base_out=self.dxn, out=self.dattn, tag="o", site=(l, 1), gW=S.gWo)
            if self.native_attn:
                self._join("qkv")  # the previous layer's qkv weight gradients read dqkv / du_qkv
                if self.nkv == nh:
                    C.attention_bwd(self.qkv[sl], self.attn_o[l], self.dattn, self.lse[l], self.delta, self.dqkv, B, T, nh, hd,
                                    1.0 / math.sqrt(hd))
                else:
                    C.attention_bwd(self.qkv[sl], self.attn_o[l], self.dattn, self.lse[l], self.delta, self.dqkv, B, T, nh, hd,
                                    1.0 / math.sqrt(hd), nkv=self.nkv)
                C.rope_inplace(self.dqkv, T, nh + self.nkv, hd, hd, self.cos, self.sin, True, 0)  # back through the rotation of q, k
                dq = None
            else:
                dq, dk, dv = self._sdpa_bwd(l)
                self._join("qkv")  # the previous layer's qkv weight gradients read dqkv / du_qkv
            if dq is None:
                pass
            elif self.nkv == nh and dq.stride() == dk.stride() == dv.stride() and dq.stride(3) == 1:
                C.rope_pack_bwd(dq, dk, dv, self.dqkv, hd, self.cos, self.sin, 0)  # gather + inverse rotation in one pass
            elif self.nkv != nh and dk.stride() == dv.stride() and dq.stride(3) == 1 and dk.stride(3) == 1:
                C.rope_pack_bwd(dq, dk, dv, self.dqkv, hd, self.cos, self.sin, 0, nkv=self.nkv)
            else:
                nkv = self.nkv
                d3 = self.dqkv.view(B, T, nh + 2 * nkv, hd)
                d3[:, :, :nh].copy_(dq.transpose(1, 2))
                d3[:, :, nh:nh + nkv].copy_(dk.transpose(1, 2))
                d3[:, :, nh + nkv:].copy_(dv.transpose(1, 2))
                C.rope_inplace(self.dqkv, T, nh + nkv, hd, hd, self.cos, self.sin, True, 0)
            self._lora_group_bwd(self.dqkv, S.B_qkv, S.Wqkv, S.A_qkv, S.gA_qkv, S.gB_qkv, self.xd_qkv[sl], self.u_qkv[sl],
                                 S.keys_qkv, G=3, K=h, Ng=self.kv, base_out=self.dxn, out=self.dxn2, tag="qkv", site=(l, 0), Nq=h,
                                 gW=S.gWqkv)
            self._join("d")  # this layer's down_proj weight gradients read the buffer written next
            C.rmsnorm_bwd(self.dxn2, self.x_in[l], S.w1, self.rstd1[sl], dx, dx_other, S.gw1, ws, tk)
            dx, dx_other = dx_other, dx
        self._embedding_bwd_and_join(dx, ("d", "gu", "o", "qkv"))
        if self.fp8_bwd:
            self._fp8_bwd_calibrated = True  # the first backward ran in bf16 and recorded the gradient amax of every site

    def _fp8_calibrate(self):
        """Bootstrap of the delayed activation scales: one bf16 forward that only *records* every site's amax.  (Starting the
        fp8 path cold would saturate the first sites, shrink everything downstream and need one pass per site to recover.)"""
        self._fp8_calibrating = True
        try:
            self.labels.view(self.B_, self.T_)[:, :-1].copy_(self.ids[:, 1:])
            self._forward(True)
        finally:
            self._fp8_calibrating = False
        self._fp8_calibrated = True

    def _fp8_prep(self):
        """Rotates the activation amax state and derives the scales of a micro-step (a training forward starts with it)."""
        self.C.fp8_prep(self._act_state2, self._w_scale2, self._inv_sx2, self._alpha_main2, self._alpha_inv2, self.fp8_margin,
                        4 * self.L)

    # ------------------------------------------------------------------ public stepper interface
    def _before_micro(self):
        if self.fp8 and not self._fp8_calibrated:
            self._fp8_calibrate()

    def _eval_body(self):
        if self.fp8 and not self._fp8_calibrated:
            # evaluation before the first training step: bootstrap the activation scales exactly like micro_step does
            self._fp8_calibrate()
            self._fp8_prep()
        super()._eval_body()

    @torch.no_grad()
    def merge_and_reinit(self):
        """The merge of every stacked block (see the base class), then the E4M3 copies of the merged weights.  Packed stacks
        (``_merge_packed``): afterwards the modules' input-gradient scales are refreshed from their stacks'."""
        super().merge_and_reinit()
        if self.fp8:
            self._quantize_weights()

    def _packed_merged(self, l: int) -> None:
        for group, st in zip(self._stack_rows(self.inner.model.layers[l]), self.Wmx[l]):
            for m, r0 in group:
                mx.refresh_part(st, m.qweight, r0)
