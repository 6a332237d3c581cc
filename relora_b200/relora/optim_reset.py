"""Optimizer-state resets performed at every ReLoRA cycle boundary.

Parity target: reference ``peft_pretraining/training_utils.py:150-170`` (the two in-place
pruning primitives) and ``:267-364`` (``optimizer_reset``).  Three mutually exclusive modes:

* ``reset_optimizer_on_relora`` — "reset" = random pruning with ratio 0.999 (the reference does
  this instead of zeroing because of a ZeRO state-dict issue; we keep the behaviour);
* ``optimizer_random_pruning=p`` — keep each element with probability ``1-p``;
* ``optimizer_magnitude_pruning=p`` — keep ``|x| > quantile(|x|, p)`` (strict inequality).

Differences by design:

* the random mask is drawn from an explicit counter-based generator keyed by
  ``(seed, reset_index, tensor_index)`` so every data-parallel rank prunes identically without
  relying on generator lock-step (SURVEY §3.3);
* the zero-count statistic is accumulated on the device and read back once, not once per tensor;
* on CUDA the flat-buffer path dispatches to the fused ``state_prune`` kernels (``ops.prune``).
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import torch

from ..obs import logger

__all__ = ["random_pruning_", "magnitude_pruning_", "magnitude_threshold", "optimizer_reset", "resolve_reset_mode"]


@torch.no_grad()
def random_pruning_(tensor: torch.Tensor, prune_ratio: float, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """Zero each element independently with probability ``prune_ratio`` (in place)."""
    keep = torch.rand(tensor.shape, device=tensor.device, dtype=torch.float32, generator=generator) > prune_ratio
    tensor.mul_(keep.to(tensor.dtype))
    return tensor


@torch.no_grad()
def magnitude_threshold(tensor: torch.Tensor, prune_ratio: float) -> torch.Tensor:
    """``quantile(|x|, q)`` with linear interpolation, computed in fp32, cast to ``tensor.dtype``.

    Implemented with two ``kthvalue`` selects instead of ``torch.quantile`` (which sorts and is
    capped at 16 M elements) — same value, no size limit.
    """
    mag = tensor.detach().abs().flatten().to(torch.float32)
    n = mag.numel()
    pos = prune_ratio * (n - 1)
    lo = int(pos)
    hi = min(lo + 1, n - 1)
    frac = pos - lo
    v_lo = torch.kthvalue(mag, lo + 1).values
    if frac > 0.0 and hi != lo:
        v_hi = torch.kthvalue(mag, hi + 1).values
        thr = torch.lerp(v_lo, v_hi, torch.tensor(frac, dtype=torch.float32, device=mag.device))
    else:
        thr = v_lo
    return thr.to(tensor.dtype)


@torch.no_grad()
def magnitude_pruning_(tensor: torch.Tensor, prune_ratio: float) -> torch.Tensor:
    """Zero every element whose magnitude is not strictly above the ``prune_ratio`` quantile."""
    thr = magnitude_threshold(tensor, prune_ratio)
    tensor.mul_((tensor.abs() > thr).to(tensor.dtype))
    return tensor


def resolve_reset_mode(reset_optimizer_on_relora: bool, optimizer_random_pruning: float, optimizer_magnitude_pruning: float):
    """Validate exclusivity and return ``(kind, ratio)`` with kind in {"random", "magnitude"}."""
    chosen = int(bool(reset_optimizer_on_relora)) + int(bool(optimizer_random_pruning)) + int(bool(optimizer_magnitude_pruning))
    if chosen != 1:
        logger.warning(
            f"Got {reset_optimizer_on_relora=}, {optimizer_random_pruning=}, {optimizer_magnitude_pruning=}"
        )
        raise ValueError(
            "Exactly one of reset_optimizer_on_relora, optimizer_random_pruning, "
            "optimizer_magnitude_pruning must be True"
        )
    if reset_optimizer_on_relora:
        return "random", 0.999
    if optimizer_random_pruning:
        return "random", float(optimizer_random_pruning)
    return "magnitude", float(optimizer_magnitude_pruning)


def _state_of(optimizer):
    """Per-parameter state mapping, looking through a ZeRO wrapper if present."""
    inner = getattr(optimizer, "optim", None)
    if inner is not None and hasattr(inner, "state") and type(optimizer).__name__ == "ZeroRedundancyOptimizer":
        return inner.state
    return optimizer.state


@torch.no_grad()
def optimizer_reset(
    optimizer,
    *,
    reset_params: Sequence[torch.nn.Parameter],
    optimizer_state_keys: Iterable[str],
    reset_optimizer_on_relora: bool,
    optimizer_random_pruning: float,
    optimizer_magnitude_pruning: float,
    seed: int = 0,
    reset_index: int = 0,
) -> float:
    """Prune the Adam moments of ``reset_params`` in place; returns the % of zeroed entries.

    Works on any ``torch.optim.Optimizer``-like object, ``ZeroRedundancyOptimizer`` and this
    repo's :class:`relora_b200.parallel.flat_optim.FlatAdamW` (which exposes ``prune_state``).
    """
    kind, ratio = resolve_reset_mode(reset_optimizer_on_relora, optimizer_random_pruning, optimizer_magnitude_pruning)
    if kind == "random":
        logger.info(f"Performing random pruning of optimizer states. Pruning {ratio} percent")
    else:
        logger.info(f"Performing magnitude pruning of optimizer states. Pruning {ratio} percent")

    if hasattr(optimizer, "prune_state"):
        pct = optimizer.prune_state(reset_params, list(optimizer_state_keys), kind, ratio, seed=seed, reset_index=reset_index)
        logger.info(f"Percent of optimizer states zeroed: {pct:.2f}")
        return pct

    state = _state_of(optimizer)
    keys: List[str] = list(optimizer_state_keys)
    n_total = 0
    n_zero = None
    for t_idx, p in enumerate(reset_params):
        pstate = state.get(p, {})
        if len(pstate) == 0:  # unsharded param under ZeRO, or a param that never got a gradient
            continue
        for k_idx, key in enumerate(keys):
            buf = pstate[key]
            if kind == "random":
                gen = torch.Generator(device=buf.device)
                gen.manual_seed((seed * 1_000_003 + reset_index) * 1_000_003 + t_idx * len(keys) + k_idx)
                random_pruning_(buf, ratio, generator=gen)
            else:
                magnitude_pruning_(buf, ratio)
            n_total += buf.numel()
            z = (buf == 0).sum()
            n_zero = z if n_zero is None else n_zero + z
    pct = float(n_zero.item()) / (1e-7 + n_total) * 100 if n_zero is not None else 0.0
    logger.info(f"Percent of optimizer states zeroed: {pct:.2f}")
    return pct
