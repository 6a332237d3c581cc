"""Data-parallel gradient synchronisation + clipping on the flat gradient buffer.

Upstream wraps the model in ``DistributedDataParallel`` and therefore all-reduces every bucket on
*every micro-batch* (no ``no_sync`` around accumulation, ``torchrun_main.py:616-622, 796-800``) and
re-broadcasts the rotary buffers on every forward.  Here the gradients of all accumulation
micro-steps are summed locally and reduced ONCE per update — mathematically identical.

Transports:

* ``nccl``  — one ``all_reduce`` (or ``reduce_scatter`` + ``all_gather`` for ZeRO-1) on the flat
  buffer: the baseline path implemented here, also used with gloo on CPU;
* ``p2p``   — :class:`relora_b200.parallel.symm.SymmComm.fused_update`: hand-written sm_90a kernels over NVLink
  peer memory / NVLS multicast (reduce-scatter + Σg² + AdamW + parameter broadcast in one chain).  The steppers
  call it directly and bypass :meth:`GradSync.reduce`; ``transport`` is then only a label.

The global gradient norm for clipping is produced here as a device scalar so that the optimizer can
consume ``clip_coef / world`` without a host synchronisation.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist

from .dist import DistInfo
from .flat import FlatParamStore

__all__ = ["GradSync", "broadcast_params"]


@torch.no_grad()
def broadcast_params(module: torch.nn.Module, src: int = 0) -> None:
    """One-time replica synchronisation (what the DDP constructor does upstream, SURVEY N4)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return
    seen = set()
    for t in list(module.parameters()) + [b for b in module.buffers()]:
        base = t.data
        if base.data_ptr() in seen:
            continue
        seen.add(base.data_ptr())
        dist.broadcast(base, src=src)
    # block-scaled frozen weights are neither parameters nor buffers (packed bytes + scales): replicate them as well
    for m in module.modules():
        qw = getattr(m, "__dict__", {}).get("qweight")
        if qw is None:
            continue
        for name in ("q", "sf_fwd", "sf_bwd", "data", "scales", "tensor_scale"):
            t = getattr(qw, name, None)
            if torch.is_tensor(t) and t.numel() > 0:
                if t.dim() == 0:
                    buf = t.reshape(1).clone()
                    dist.broadcast(buf, src=src)
                    t.copy_(buf[0])
                else:
                    dist.broadcast(t, src=src)


class GradSync:
    def __init__(self, store: FlatParamStore, info: DistInfo, *, transport: str = "nccl", zero: bool = False):
        self.store, self.info, self.zero = store, info, zero
        self.world = info.world_size
        self.transport = transport if self.world > 1 else "none"
        if zero and self.world > 1:
            self.shard = store.shard_bounds(info.rank, self.world)
        else:
            self.shard = (0, store.numel)

    @torch.no_grad()
    def reduce(self) -> None:
        """Sum gradients across ranks (full buffer, or own shard under ZeRO-1)."""
        if self.world == 1:
            return
        g = self.store.grads
        if self.zero:
            lo, hi = self.shard
            dist.reduce_scatter_tensor(g[lo:hi], g, op=dist.ReduceOp.SUM)
        else:
            dist.all_reduce(g, op=dist.ReduceOp.SUM)

    @torch.no_grad()
    def gather_params(self) -> None:
        """ZeRO-1: publish the updated parameter shards to every replica."""
        if self.world == 1 or not self.zero:
            return
        lo, hi = self.shard
        p = self.store.params
        dist.all_gather_into_tensor(p, p[lo:hi].clone())

    @torch.no_grad()
    def grad_norm_and_scale(self, max_norm: float) -> Tuple[torch.Tensor, torch.Tensor]:
        """Return ``(total_norm, grad_scale)`` as device scalars.

        ``total_norm`` is the 2-norm of the world-averaged gradient (what ``clip_grad_norm_``
        reports upstream after DDP averaging); ``grad_scale = clip_coef / world``.
        """
        lo, hi = self.shard
        g = self.store.grads[lo:hi]
        sq = g.to(torch.float32).pow(2).sum() if not g.is_cuda else torch.linalg.vector_norm(g, 2, dtype=torch.float32).pow(2)
        if self.zero and self.world > 1:
            dist.all_reduce(sq, op=dist.ReduceOp.SUM)
        total = sq.sqrt() / self.world
        if max_norm and max_norm > 0:
            coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
        else:
            coef = torch.ones_like(total)
        # a non-finite norm poisons the scale: the optimizer skips the update instead of writing NaNs into the parameters
        coef = torch.where(torch.isfinite(total), coef, torch.full_like(coef, float("nan")))
        return total, coef / self.world
