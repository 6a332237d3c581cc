"""Llama decoder-only language model with HF-compatible parameter names.

Parity target: reference ``peft_pretraining/modeling_llama.py`` (RMSNorm ``:74-91``, rotary tables
``:94-141``, SwiGLU MLP ``:144-158``, causal SDPA attention that ignores the padding mask
``:161-240``, pre-norm residual block ``:243-308``, N(0, 0.02) init ``:339-348``, shifted
cross-entropy ``:694-708``, sequence classification head ``:775-879``).

This is a plain ``nn.Module`` tree (no ``PreTrainedModel`` machinery); ``save_pretrained`` /
``from_pretrained`` read and write the reference checkpoint layout (``config.json`` +
``pytorch_model.bin``).  State-dict keys match the reference exactly, including the persistent
``rotary_emb.inv_freq`` buffers, so checkpoints are interchangeable in both directions.

Two execution paths share these parameters:

* the module-by-module path below (PyTorch expressions; on CUDA/bf16 the leaf modules dispatch to
  the native kernels through :mod:`relora_b200.ops.dispatch`);
* the whole-layer fused executor in :mod:`relora_b200.engine.fused_llama`, which the trainer uses on
  H100 (stacked QKV / gate-up weights, LoRA folded into the GEMM, CUDA-graph captured).
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .configs import load_config, save_config

__all__ = [
    "LlamaRMSNorm",
    "LlamaRotaryEmbedding",
    "LlamaMLP",
    "LlamaAttention",
    "LlamaDecoderLayer",
    "LlamaModel",
    "LlamaForCausalLM",
    "LlamaForSequenceClassification",
    "CausalLMOutput",
    "SequenceClassifierOutput",
    "rotate_half",
    "apply_rotary_pos_emb",
]


class _Output(dict):
    """Dict with attribute access (stands in for HF ``ModelOutput``; works with HF ``Trainer``)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None

    def __setattr__(self, k, v):
        self[k] = v

    def to_tuple(self):
        return tuple(v for v in self.values() if v is not None)

    def __getitem__(self, k):
        if isinstance(k, int):
            return self.to_tuple()[k]
        return super().__getitem__(k)


class CausalLMOutput(_Output):
    pass


class SequenceClassifierOutput(_Output):
    pass


# --------------------------------------------------------------------------- building blocks
class LlamaRMSNorm(nn.Module):
    """y = weight * bf16(x * rsqrt(mean(x²) + eps)) — normalise in fp32, round, then scale."""

    def __init__(self, hidden_size: int, eps: float = 1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        from ..ops import dispatch

        if dispatch.use_fused(x):
            from ..ops import fused

            return fused.rmsnorm(x, self.weight, self.variance_epsilon)
        var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
        y = x * torch.rsqrt(var + self.variance_epsilon)
        if self.weight.dtype in (torch.float16, torch.bfloat16):
            y = y.to(self.weight.dtype)
        return self.weight * y


class LlamaRotaryEmbedding(nn.Module):
    """cos/sin tables in the half-rotation layout; built in fp32, cast with the module."""

    def __init__(self, dim: int, max_position_embeddings: int = 2048, base: float = 10000.0, device=None):
        super().__init__()
        self.dim = dim
        self.base = base
        inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.float32, device=device) / dim))
        self.register_buffer("inv_freq", inv_freq)  # persistent: appears in reference checkpoints
        self._build(max_position_embeddings, inv_freq)

    def _build(self, n: int, inv_freq: torch.Tensor):
        self.max_seq_len_cached = n
        t = torch.arange(n, device=inv_freq.device, dtype=inv_freq.dtype)
        freqs = torch.outer(t, inv_freq)
        emb = torch.cat((freqs, freqs), dim=-1)
        self.register_buffer("cos_cached", emb.cos()[None, None], persistent=False)
        self.register_buffer("sin_cached", emb.sin()[None, None], persistent=False)

    def forward(self, x, seq_len: int):
        if seq_len > self.max_seq_len_cached:
            self._build(seq_len, self.inv_freq.to(x.device))
        return (
            self.cos_cached[:, :, :seq_len].to(dtype=x.dtype),
            self.sin_cached[:, :, :seq_len].to(dtype=x.dtype),
        )


def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def apply_rotary_pos_emb(q, k, cos, sin, position_ids):
    cos = cos[0, 0][position_ids].unsqueeze(1)  # [B, 1, T, hd]
    sin = sin[0, 0][position_ids].unsqueeze(1)
    return (q * cos) + (rotate_half(q) * sin), (k * cos) + (rotate_half(k) * sin)


class LlamaMLP(nn.Module):
    def __init__(self, hidden_size: int, intermediate_size: int, hidden_act: str = "silu"):
        super().__init__()
        if hidden_act != "silu":
            raise NotImplementedError(f"hidden_act={hidden_act}: Llama configs here use silu")
        self.gate_proj = nn.Linear(hidden_size, intermediate_size, bias=False)
        self.down_proj = nn.Linear(intermediate_size, hidden_size, bias=False)
        self.up_proj = nn.Linear(hidden_size, intermediate_size, bias=False)

    def forward(self, x):
        return self.down_proj(F.silu(self.gate_proj(x)) * self.up_proj(x))


class LlamaAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.num_heads = config.num_attention_heads
        self.head_dim = self.hidden_size // self.num_heads
        if self.head_dim * self.num_heads != self.hidden_size:
            raise ValueError(
                f"hidden_size must be divisible by num_heads (got `hidden_size`: {self.hidden_size}"
                f" and `num_heads`: {self.num_heads})."
            )
        self.max_position_embeddings = config.max_position_embeddings
        self.q_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self.k_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self.v_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self.o_proj = nn.Linear(self.hidden_size, self.hidden_size, bias=False)
        self.rotary_emb = LlamaRotaryEmbedding(self.head_dim, max_position_embeddings=self.max_position_embeddings)

    def forward(self, hidden_states, position_ids=None, past_key_value=None, use_cache=False):
        B, T, _ = hidden_states.shape
        q = self.q_proj(hidden_states).view(B, T, self.num_heads, self.head_dim).transpose(1, 2)
        k = self.k_proj(hidden_states).view(B, T, self.num_heads, self.head_dim).transpose(1, 2)
        v = self.v_proj(hidden_states).view(B, T, self.num_heads, self.head_dim).transpose(1, 2)
        kv_len = T + (past_key_value[0].shape[-2] if past_key_value is not None else 0)
        cos, sin = self.rotary_emb(v, seq_len=kv_len)
        q, k = apply_rotary_pos_emb(q, k, cos, sin, position_ids)
        if past_key_value is not None:
            k = torch.cat([past_key_value[0], k], dim=2)
            v = torch.cat([past_key_value[1], v], dim=2)
        present = (k, v) if use_cache else None
        # the padding mask is ignored and causality always applied (reference :221-224)
        causal = past_key_value is None or T > 1
        if past_key_value is not None and T > 1:
            # chunked prefill onto a cache: lower-right aligned causal mask
            mask = torch.ones(T, kv_len, dtype=torch.bool, device=q.device).tril(diagonal=kv_len - T)
            out = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        elif causal and past_key_value is None and _use_native_attention(q, self.head_dim):
            # this repo's wgmma flash-attention kernels (csrc/attention.cu) instead of the library SDPA call
            from ..ops import fused

            out = fused.causal_attention(q, k, v)
        else:
            out = F.scaled_dot_product_attention(q, k, v, dropout_p=0.0, is_causal=causal)
        out = out.transpose(1, 2).reshape(B, T, self.hidden_size)
        return self.o_proj(out), present


def _use_native_attention(q: torch.Tensor, head_dim: int) -> bool:
    """CUDA + bf16 + head_dim <= 64 (multiple of 8): the wgmma kernels; RELORA_B200_ATTENTION=sdpa forces the library call."""
    if not q.is_cuda or os.environ.get("RELORA_B200_ATTENTION", "auto") == "sdpa":
        return False
    from ..ops import dispatch, fused

    return dispatch.use_fused(q) and fused.native_attention_supported(q, head_dim)


class LlamaDecoderLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.self_attn = LlamaAttention(config)
        self.mlp = LlamaMLP(config.hidden_size, config.intermediate_size, getattr(config, "hidden_act", "silu"))
        self.input_layernorm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.post_attention_layernorm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)

    def forward(self, hidden_states, position_ids=None, past_key_value=None, use_cache=False):
        residual = hidden_states
        h, present = self.self_attn(self.input_layernorm(hidden_states), position_ids, past_key_value, use_cache)
        hidden_states = residual + h
        residual = hidden_states
        hidden_states = residual + self.mlp(self.post_attention_layernorm(hidden_states))
        return hidden_states, present


# --------------------------------------------------------------------------- base classes
class _PretrainedMixin:
    """``save_pretrained`` / ``from_pretrained`` in the reference layout."""

    config_class_name = "LlamaConfig"

    def _init_weights(self, module):
        std = getattr(self.config, "initializer_range", 0.02)
        if isinstance(module, nn.Linear):
            module.weight.data.normal_(mean=0.0, std=std)
            if module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.Embedding):
            module.weight.data.normal_(mean=0.0, std=std)
            if module.padding_idx is not None:
                module.weight.data[module.padding_idx].zero_()

    def post_init(self):
        self.apply(self._init_weights)

    def save_pretrained(self, path: str, safe_serialization: bool = False, **_):
        os.makedirs(path, exist_ok=True)
        save_config(self.config, path)
        state = {k: v.detach().cpu() for k, v in self.state_dict().items()}
        torch.save(state, os.path.join(path, "pytorch_model.bin"))  # readers hard-code this name
        if safe_serialization:
            try:
                from safetensors.torch import save_file

                save_file({k: v.contiguous() for k, v in state.items()}, os.path.join(path, "model.safetensors"))
            except Exception:  # pragma: no cover
                pass

    @classmethod
    def from_pretrained(cls, path: str, **kwargs):
        config = load_config(path)
        model = cls(config, **kwargs)
        bin_path = os.path.join(path, "pytorch_model.bin")
        if os.path.exists(bin_path):
            state = torch.load(bin_path, map_location="cpu", weights_only=True)
        else:
            from safetensors.torch import load_file

            state = load_file(os.path.join(path, "model.safetensors"))
        model.load_state_dict(state, strict=True)
        return model

    def num_parameters(self, only_trainable: bool = False) -> int:
        return sum(p.numel() for p in self.parameters() if p.requires_grad or not only_trainable)

    def gradient_checkpointing_enable(self, **_):
        for m in self.modules():
            if hasattr(m, "gradient_checkpointing"):
                m.gradient_checkpointing = True

    def gradient_checkpointing_disable(self):
        for m in self.modules():
            if hasattr(m, "gradient_checkpointing"):
                m.gradient_checkpointing = False


class LlamaModel(nn.Module, _PretrainedMixin):
    def __init__(self, config):
        super().__init__()
        self.config = config
        pad = getattr(config, "pad_token_id", None)
        self.padding_idx = pad
        self.vocab_size = config.vocab_size
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, padding_idx=pad)
        self.layers = nn.ModuleList([LlamaDecoderLayer(config) for _ in range(config.num_hidden_layers)])
        self.norm = LlamaRMSNorm(config.hidden_size, eps=config.rms_norm_eps)
        self.gradient_checkpointing = False

    def get_input_embeddings(self):
        return self.embed_tokens

    def set_input_embeddings(self, value):
        self.embed_tokens = value

    def forward(
        self,
        input_ids=None,
        attention_mask=None,  # accepted, ignored by attention exactly like the reference
        position_ids=None,
        past_key_values: Optional[List[Tuple[torch.Tensor, torch.Tensor]]] = None,
        inputs_embeds=None,
        use_cache: Optional[bool] = None,
        output_hidden_states: bool = False,
    ):
        if (input_ids is None) == (inputs_embeds is None):
            raise ValueError("You have to specify exactly one of input_ids or inputs_embeds")
        if inputs_embeds is None:
            inputs_embeds = self.embed_tokens(input_ids)
        B, T, _ = inputs_embeds.shape
        past_len = past_key_values[0][0].shape[2] if past_key_values is not None else 0
        if position_ids is None:
            position_ids = torch.arange(past_len, past_len + T, dtype=torch.long, device=inputs_embeds.device)
            position_ids = position_ids.unsqueeze(0).expand(B, T)
        else:
            position_ids = position_ids.view(-1, T).long()
        use_cache = bool(use_cache) and not (self.gradient_checkpointing and self.training)

        h = inputs_embeds
        all_h = [] if output_hidden_states else None
        cache = [] if use_cache else None
        for i, layer in enumerate(self.layers):
            if all_h is not None:
                all_h.append(h)
            past = past_key_values[i] if past_key_values is not None else None
            if self.gradient_checkpointing and self.training:
                h, present = torch.utils.checkpoint.checkpoint(layer, h, position_ids, None, False, use_reentrant=False)
            else:
                h, present = layer(h, position_ids, past, use_cache)
            if cache is not None:
                cache.append(present)
        h = self.norm(h)
        if all_h is not None:
            all_h.append(h)
        return h, cache, all_h


class LlamaForCausalLM(nn.Module, _PretrainedMixin):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.model = LlamaModel(config)
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        self.post_init()

    # HF-style accessors
    def get_input_embeddings(self):
        return self.model.embed_tokens

    def set_input_embeddings(self, value):
        self.model.embed_tokens = value

    def get_output_embeddings(self):
        return self.lm_head

    def set_output_embeddings(self, new):
        self.lm_head = new

    def get_decoder(self):
        return self.model

    def forward(
        self,
        input_ids=None,
        attention_mask=None,
        position_ids=None,
        past_key_values=None,
        inputs_embeds=None,
        labels=None,
        use_cache=None,
        output_attentions=None,
        output_hidden_states=None,
        return_dict=None,
        return_logits: bool = True,
    ):
        h, cache, all_h = self.model(
            input_ids=input_ids,
            attention_mask=attention_mask,
            position_ids=position_ids,
            past_key_values=past_key_values,
            inputs_embeds=inputs_embeds,
            use_cache=use_cache,
            output_hidden_states=bool(output_hidden_states),
        )
        loss = None
        logits = None
        if labels is not None and not return_logits:
            from ..ops import reference as _ref, dispatch

            if dispatch.use_fused(h):
                from ..ops import fused

                loss = fused.lm_head_cross_entropy(h, self.lm_head.weight, labels)
            else:
                loss = _ref.lm_head_cross_entropy(h, self.lm_head.weight, labels)
        else:
            logits = self.lm_head(h)
            if labels is not None:
                shift_logits = logits[..., :-1, :].contiguous()
                shift_labels = labels[..., 1:].contiguous().to(shift_logits.device)
                loss = F.cross_entropy(shift_logits.view(-1, self.config.vocab_size), shift_labels.view(-1))
        return CausalLMOutput(loss=loss, logits=logits, past_key_values=cache, hidden_states=all_h, attentions=None)

    @torch.no_grad()
    def generate(self, input_ids, max_new_tokens: int = 20, eos_token_id: Optional[int] = None, do_sample: bool = False, temperature: float = 1.0):
        """Greedy / temperature sampling with a KV cache (the reference gets this from HF ``generate``)."""
        out = self(input_ids=input_ids, use_cache=True)
        cache = out.past_key_values
        tokens = input_ids
        nxt_logits = out.logits[:, -1]
        for _ in range(max_new_tokens):
            if do_sample:
                nxt = torch.multinomial(torch.softmax(nxt_logits.float() / temperature, -1), 1)
            else:
                nxt = nxt_logits.argmax(-1, keepdim=True)
            tokens = torch.cat([tokens, nxt], dim=1)
            if eos_token_id is not None and bool((nxt == eos_token_id).all()):
                break
            out = self(input_ids=nxt, past_key_values=cache, use_cache=True)
            cache = out.past_key_values
            nxt_logits = out.logits[:, -1]
        return tokens


class LlamaForSequenceClassification(nn.Module, _PretrainedMixin):
    """Llama trunk + linear ``score`` head on the last non-pad token (reference ``:775-879``)."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.num_labels = getattr(config, "num_labels", 2)
        self.model = LlamaModel(config)
        self.score = nn.Linear(config.hidden_size, self.num_labels, bias=False)
        self.post_init()

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def set_input_embeddings(self, value):
        self.model.embed_tokens = value

    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, labels=None, use_cache=None, output_attentions=None,
                output_hidden_states=None, return_dict=None):
        h, cache, all_h = self.model(
            input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
            past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
            output_hidden_states=bool(output_hidden_states),
        )
        logits = self.score(h)
        B = logits.shape[0]
        pad = getattr(self.config, "pad_token_id", None)
        if pad is None and B != 1:
            raise ValueError("Cannot handle batch sizes > 1 if no padding token is defined.")
        if pad is None or input_ids is None:
            last = torch.full((B,), -1, device=logits.device, dtype=torch.long)
        else:
            # index of the last token before the first pad (wraps to -1 when there is no pad)
            last = (torch.ne(input_ids, pad).sum(-1) - 1).to(logits.device)
        pooled = logits[torch.arange(B, device=logits.device), last]

        loss = None
        if labels is not None:
            labels = labels.to(pooled.device)
            ptype = getattr(self.config, "problem_type", None)
            if ptype is None:
                if self.num_labels == 1:
                    ptype = "regression"
                elif labels.dtype in (torch.long, torch.int):
                    ptype = "single_label_classification"
                else:
                    ptype = "multi_label_classification"
                self.config.problem_type = ptype
            if ptype == "regression":
                loss = F.mse_loss(pooled.squeeze(), labels.squeeze()) if self.num_labels == 1 else F.mse_loss(pooled, labels)
            elif ptype == "single_label_classification":
                loss = F.cross_entropy(pooled.view(-1, self.num_labels), labels.view(-1))
            else:
                loss = F.binary_cross_entropy_with_logits(pooled, labels)
        return SequenceClassifierOutput(loss=loss, logits=pooled, past_key_values=cache, hidden_states=all_h, attentions=None)
