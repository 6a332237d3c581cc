"""``ReLoRaLinear`` — a frozen linear layer plus a trainable low-rank branch.

    y = x Wᵀ + b + s · B(A(dropout(x)))        s = alpha / r   (or tanh(scaling) if trainable)

Parity target: reference ``peft_pretraining/relora.py:181-323``.  Parameter names are the
reference's (``weight``, ``bias``, ``lora_A.weight`` [r, in], ``lora_B.weight`` [out, r],
``scaling``) so checkpoints interchange.  What is different here:

* the frozen weight may be stored block-scaled (``mxfp8`` / ``nvfp4``; ``8bit`` / ``4bit`` are
  aliases) instead of bitsandbytes NF4 / int8, and the 8-bit merge works (it is broken upstream);
* the merge accumulates ``W += s·B@A`` in fp32 before rounding back to the storage dtype;
* re-initialisation of ``A`` draws from a counter-based generator keyed by
  ``(seed, restart_index, module_index)`` so all data-parallel ranks agree by construction;
* on CUDA the forward/backward dispatches to the fused sm_90a kernels in :mod:`relora_b200.ops`
  (one pass over ``x`` for frozen + low-rank branch); the PyTorch expression below is the
  reference implementation used on CPU and for numerics tests.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..obs import logger
from ..ops import quant as _quant

__all__ = ["ReLoRaLinear", "kaiming_bound", "packed_linear"]


def kaiming_bound(fan_in: int, a: float = math.sqrt(5)) -> float:
    """Half-width of ``kaiming_uniform_(a)``: gain·sqrt(3/fan_in) with gain = sqrt(2/(1+a²))."""
    gain = math.sqrt(2.0 / (1.0 + a * a))
    return gain * math.sqrt(3.0 / fan_in)


class _Factor(nn.Module):
    """A bias-free linear map that owns ``weight`` — keeps the ``lora_A.weight`` key layout."""

    def __init__(self, in_features: int, out_features: int, device=None, dtype=None):
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features, device=device, dtype=dtype))
        self.bias = None

    def forward(self, x):
        return F.linear(x, self.weight)

    def extra_repr(self):
        return f"in_features={self.in_features}, out_features={self.out_features}, bias=False"


class ReLoRaLinear(nn.Module):
    def __init__(
        self,
        in_features: int,
        out_features: int,
        r: int,
        *,
        lora_alpha: float = 1,
        lora_dropout: float = 0.1,
        lora_only: bool = False,
        weight_data: Optional[torch.Tensor] = None,
        bias_data: Optional[torch.Tensor] = None,
        trainable_scaling: bool = False,
        bias: bool = True,
        device=None,
        dtype=None,
        quantize=None,
        bnb_4bit_use_double_quant: bool = False,  # accepted for CLI parity; block scales have no second level
        bnb_4bit_quant_type: str = "nf4",
    ):
        super().__init__()
        if r <= 0:
            raise ValueError("r must be positive. If you want r == 0, use the original model.")
        self.in_features = in_features
        self.out_features = out_features
        self.r = r
        self.lora_alpha = lora_alpha
        self.lora_dropout = nn.Dropout(p=lora_dropout)
        self.lora_only = lora_only
        self.trainable_scaling = trainable_scaling
        self.quantize = _quant.canonical_format(quantize)
        self.qweight: Optional[_quant.QuantizedWeight] = None
        self.module_index = 0  # set by ReLoRaModel; keys the re-init RNG stream

        if lora_only:
            self.weight = None
            self.bias = None
        else:
            if bias:
                if bias_data is None:
                    bias_data = torch.zeros(out_features, device=device, dtype=dtype)
                self.bias = nn.Parameter(bias_data)
            else:
                self.bias = None
            if weight_data is None:
                weight_data = torch.zeros(out_features, in_features, device=device, dtype=dtype)
            if self.quantize is None:
                self.weight = nn.Parameter(weight_data, requires_grad=False)
            else:
                # ONLY the packed bytes + block scales are resident (like bitsandbytes' Params4bit / Int8Params upstream,
                # relora.py:224-236): `self.weight` is no parameter but a transient dequantised view (see __getattr__), the
                # forward / backward dequantise one layer at a time, and state_dict() still carries a `weight` entry so that
                # checkpoints keep the reference layout
                self._wdtype = weight_data.dtype
                self.qweight = _quant.quantize(weight_data, self.quantize)

        self.lora_A = _Factor(in_features, r, device=device, dtype=dtype)
        self.lora_B = _Factor(r, out_features, device=device, dtype=dtype)
        nn.init.kaiming_uniform_(self.lora_A.weight, a=math.sqrt(5))
        nn.init.zeros_(self.lora_B.weight)
        if trainable_scaling:
            self.scaling = nn.Parameter(torch.tensor([1.0], device=device), requires_grad=True)
        else:
            self.scaling = self.lora_alpha / self.r

    # ------------------------------------------------------------------ helpers
    def _post_lora_scale(self):
        if self.trainable_scaling:
            return self.scaling.tanh()
        return self.scaling

    def scale_value(self) -> float:
        s = self._post_lora_scale()
        return float(s) if not torch.is_tensor(s) else float(s.detach().float().item())

    # ---- packed storage plumbing -------------------------------------------------------------------------------------
    def __getattr__(self, name):
        if name == "weight":
            qw = self.__dict__.get("qweight")
            if qw is not None:  # transient bf16 / fp32 view of the packed weight (never stored)
                return _dequantize_any(qw, self.__dict__.get("_wdtype", torch.float32))
        return super().__getattr__(name)

    def _pack(self, value: torch.Tensor):
        """Packed form of ``value``: on CUDA, ``mxfp8`` uses the tensor-core layout of csrc/gemm_mx.cu (E4M3 + one UE8M0 scale per
        32 x 32 tile, read by the e4m3 wgmma MX GEMM in forward and input gradient); everything else (CPU, nvfp4) the
        reference layout of ops/quant.py."""
        if self.quantize == "mxfp8" and value.is_cuda:
            from ..ops import mx, native

            if native.available() and mx.supported(self.out_features, self.in_features):
                return mx.quantize_weight(value.detach())
        return _quant.quantize(value.detach(), self.quantize)

    def set_weight(self, value: torch.Tensor) -> None:
        """Replace the frozen weight (merge, checkpoint load): re-packs when the storage is quantised."""
        if self.quantize is not None:
            self.qweight = self._pack(value)
        else:
            self.weight.data.copy_(value.to(self.weight.dtype))

    def frozen_weight_nbytes(self) -> int:
        """Resident bytes of the frozen weight (packed data + scales, or the dense tensor)."""
        if self.quantize is not None:
            return int(self.qweight.nbytes)
        return 0 if self.weight is None else int(self.weight.numel() * self.weight.element_size())

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        super()._save_to_state_dict(destination, prefix, keep_vars)
        if self.quantize is not None and self.qweight is not None:
            destination[prefix + "weight"] = self.weight  # dequantised: checkpoints keep the reference key / dtype

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        key = prefix + "weight"
        if self.quantize is not None and key in state_dict:
            w = state_dict.pop(key)  # not a registered parameter: consume it here
            try:
                if tuple(w.shape) != (self.out_features, self.in_features):
                    error_msgs.append(f"size mismatch for {key}: {tuple(w.shape)} vs {(self.out_features, self.in_features)}")
                else:
                    dev = _device_of(self.qweight)
                    self.qweight = self._pack(w.to(dev))
                super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)
            finally:
                state_dict[key] = w
            if key in unexpected_keys:
                unexpected_keys.remove(key)
            return
        if self.quantize is not None and strict:
            missing_keys.append(key)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    def _apply(self, fn, recurse=True):
        out = super()._apply(fn, recurse)
        if self.qweight is not None:
            cur = _device_of(self.qweight)
            probe = fn(torch.empty(0, dtype=self._wdtype, device=cur))  # where / what dtype do parameters go?
            self._wdtype = probe.dtype if probe.is_floating_point() else self._wdtype
            if probe.device != cur:
                if probe.device.type != cur.type:
                    # CPU <-> CUDA: the packed layout changes with the device (reference layout vs tensor-core layout), so re-pack
                    # from the dequantised values once (a one-time requantisation, not a per-step cost)
                    self.qweight = self._pack(_dequantize_any(self.qweight, torch.float32).to(probe.device))
                else:
                    self.qweight = self.qweight.to(probe.device)
        return out

    # ------------------------------------------------------------------ merge
    @torch.no_grad()
    def merge_and_reinit(self, *, seed: int = 0, restart_index: int = 0, generator: Optional[torch.Generator] = None):
        """``W += s·B@A`` (fp32 accumulate), then ``A ~ U(-1/sqrt(in), 1/sqrt(in))``, ``B = 0``.

        Reference: ``relora.py:269-307``.  For quantised storage the merge is
        dequantise → add → requantise with fresh block scales.
        """
        if self.lora_only:
            print("WARNING: Skipping merge and reinit, because only lora parameters are used")
            return
        scale = self._post_lora_scale()
        if torch.is_tensor(scale):
            scale = scale.to(torch.float32)
        delta = (self.lora_B.weight.to(torch.float32) @ self.lora_A.weight.to(torch.float32)) * scale
        if self.quantize is not None:
            # dequantise -> fp32 add -> requantise with fresh block scales (relora.py:277-299; the 8-bit branch is broken upstream)
            if not isinstance(self.qweight, _quant.QuantizedWeight):
                from ..ops import mx

                mx.merge_(self.qweight, delta)  # one kernel, in place on the packed bytes
            else:
                merged = _quant.dequantize(self.qweight, torch.float32) + delta
                self.qweight = _quant.quantize(merged, self.quantize)
        else:
            merged = self.weight.data.to(torch.float32) + delta
            self.weight.data.copy_(merged.to(self.weight.dtype))
        self.reinit_lora(seed=seed, restart_index=restart_index, generator=generator)

    @torch.no_grad()
    def reinit_lora(self, *, seed: int = 0, restart_index: int = 0, generator: Optional[torch.Generator] = None):
        a = self.lora_A.weight
        if generator is None:
            generator = torch.Generator(device=a.device)
            generator.manual_seed(((seed * 1_000_003 + restart_index) * 1_000_003 + self.module_index) & 0x7FFF_FFFF_FFFF_FFFF)
        bound = kaiming_bound(self.in_features)
        fresh = torch.empty(a.shape, device=a.device, dtype=torch.float32).uniform_(-bound, bound, generator=generator)
        a.copy_(fresh.to(a.dtype))
        self.lora_B.weight.zero_()
        if self.trainable_scaling:
            self.scaling.zero_()

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor):
        from ..ops import dispatch

        if dispatch.use_fused(x):
            return dispatch.lora_linear(self, x)
        if self.lora_only:
            return self.lora_B(self.lora_A(self.lora_dropout(x))) * self._post_lora_scale()
        if self.quantize is not None:
            result = packed_linear(x, self.qweight, self.bias)
        else:
            result = F.linear(x, self.weight, bias=self.bias)
        result = result + self.lora_B(self.lora_A(self.lora_dropout(x))) * self._post_lora_scale()
        return result

    def extra_repr(self):
        q = f", quantize={self.quantize}" if self.quantize else ""
        return (
            f"in_features={self.in_features}, out_features={self.out_features}, r={self.r}, "
            f"alpha={self.lora_alpha}, lora_only={self.lora_only}{q}"
        )


def _device_of(qw) -> torch.device:
    return (qw.data if isinstance(qw, _quant.QuantizedWeight) else qw.q).device


def _dequantize_any(qw, dtype) -> torch.Tensor:
    if isinstance(qw, _quant.QuantizedWeight):
        return _quant.dequantize(qw, dtype)
    from ..ops import mx

    return mx.dequantize_weight(qw, dtype)


class _PackedLinearFn(torch.autograd.Function):
    """``y = x · dequant(W)ᵀ`` for a frozen block-scaled weight.  Neither forward nor backward keeps the dequantised matrix:
    each builds the transient dense copy of ONE layer and drops it, so the resident frozen-weight memory is the packed size
    (upstream: ``bnb.matmul_4bit`` / ``bnb.matmul`` on Params4bit / Int8Params, relora.py:314-317)."""

    @staticmethod
    def forward(ctx, x, qweight):
        ctx.qweight = qweight
        return F.linear(x, _quant.dequantize(qweight, x.dtype))

    @staticmethod
    def backward(ctx, dy):
        return dy @ _quant.dequantize(ctx.qweight, dy.dtype), None


def packed_linear(x: torch.Tensor, qweight, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    if not isinstance(qweight, _quant.QuantizedWeight):
        from ..ops import mx

        return mx.linear(x, qweight, bias)  # block-scaled tensor-core GEMMs on the packed bytes (forward and input gradient)
    y = _PackedLinearFn.apply(x, qweight)
    return y if bias is None else y + bias


def _warn_once(msg, _seen=set()):
    if msg not in _seen:
        _seen.add(msg)
        logger.warning(msg)
