"""Run-time selection between the PyTorch reference ops and the native sm_90a kernels.

Policy: tensors on a CUDA device in bf16 take the native path.  If the process is on a CUDA box and
the extension cannot be loaded this raises instead of silently falling back (a silent eager fallback
would make GPU tests pass without exercising any of our kernels).  ``RELORA_B200_FORCE_REFERENCE=1``
forces the PyTorch path everywhere (used by parity tests).
"""
from __future__ import annotations

import os
from typing import Sequence

import torch

_FORCE_REF = os.environ.get("RELORA_B200_FORCE_REFERENCE", "0") == "1"
_module_level_fused = True  # module-by-module fused path (ReLoRaLinear.forward etc.)


def force_reference(flag: bool = True) -> None:
    global _FORCE_REF
    _FORCE_REF = flag


def reference_forced() -> bool:
    return _FORCE_REF


def native_available() -> bool:
    from . import native

    return native.available()


def use_fused(x: torch.Tensor) -> bool:
    """True when ``x`` should go through the native kernels."""
    if _FORCE_REF or not x.is_cuda or x.dtype != torch.bfloat16:
        return False
    from . import native

    native.require()  # raises on a CUDA box without the extension
    return _module_level_fused


def lora_linear(module, x: torch.Tensor) -> torch.Tensor:
    from . import fused

    return fused.relora_linear_module(module, x)


def merge_all(modules: Sequence, *, seed: int, restart_index: int) -> bool:
    """Batched merge+reinit on the device; returns False when the caller should loop in PyTorch."""
    if _FORCE_REF or not modules:
        return False
    w = modules[0].lora_A.weight
    if not w.is_cuda or w.dtype != torch.bfloat16:
        return False
    from . import fused, native

    native.require()
    return fused.merge_and_reinit_modules(modules, seed=seed, restart_index=restart_index)
