"""Data-parallel gradient synchronisation + clipping on the flat gradient buffer.

Upstream wraps the model in ``DistributedDataParallel`` and therefore all-reduces every bucket on
*every micro-batch* (no ``no_sync`` around accumulation, ``torchrun_main.py:616-622, 796-800``) and
re-broadcasts the rotary buffers on every forward.  Here the gradients of all accumulation
micro-steps are summed locally and reduced ONCE per update — mathematically identical.

Transports:

* ``nccl``  — one ``all_reduce`` (or ``reduce_scatter`` + ``all_gather`` for ZeRO-1) on the flat
  buffer: the baseline path implemented here, also used with gloo on CPU;
* ``p2p``   — :class:`relora_b200.parallel.symm.SymmComm.fused_update`: hand-written sm_90a kernels over NVLink
  peer memory / NVLS multicast (reduce-scatter + Σg² + AdamW + parameter broadcast in one chain), chosen by
  :func:`peer_transport` and run by :meth:`GradSync.update` in place of ``reduce`` / ``gather_params``.

:class:`GradSync` owns the whole policy -- how gradients of the flat store get from every rank into one optimizer step -- for
the module stepper and the fused executors alike: the transport's buffers, the ZeRO-1 shard and ``update()``.

The global gradient norm for clipping is produced here as a device scalar so that the optimizer can
consume ``clip_coef / world`` without a host synchronisation.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.distributed as dist

from ..ops import native
from . import symm
from .dist import DistInfo
from .flat import FlatParamStore

__all__ = ["GradSync", "UpdateInfo", "broadcast_params", "peer_transport"]


@dataclass
class UpdateInfo:
    grad_norm: torch.Tensor  # device scalar (norm of the averaged gradient, before clipping)
    # set by the peer-memory update when the caller handed it this rank's loss: mean loss over ranks and the number of ranks that
    # asked to skip (device scalars; the reference's loss_info all-reduce folded into the kernel chain, torchrun_main.py:810)
    mean_loss: Optional[torch.Tensor] = None
    skip_count: Optional[torch.Tensor] = None


def peer_transport(info: DistInfo, transport: str, eligible: bool = True):
    """The ``SymmComm`` of the hand-written NVLink update (csrc/comm.cu) when ``transport`` (``p2p`` / ``auto``) asks for it, there
    is more than one rank and symmetric memory is available; None for NCCL / gloo.  ``eligible``: the caller's parameters can live
    in symmetric memory (bf16 on CUDA).  ``p2p`` raises where ``auto`` falls back."""
    if info.world_size == 1 or transport not in ("p2p", "auto"):
        return None
    if not eligible:
        if transport == "p2p":
            raise RuntimeError("--comm p2p needs bf16 parameters on CUDA")
        return None
    if symm.symmetric_memory_available():
        try:
            return symm.SymmComm()
        except Exception as e:  # no P2P access, allocation failure, ...
            if transport == "p2p":
                raise
            from ..obs import logger

            logger.warning(f"peer-memory collectives unavailable ({type(e).__name__}: {e}); using NCCL")
    elif transport == "p2p":
        raise RuntimeError("--comm p2p needs torch symmetric memory over an NCCL process group")
    return None


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
    def __init__(self, store: FlatParamStore, info: DistInfo, *, transport: str = "nccl", zero: bool = False, comm=None,
                 stage_bf16: bool = False):
        """``comm``: what :func:`peer_transport` returned; ``store`` must then have been carved out of ``comm.allocator()``.
        ``stage_bf16``: the store's gradients are fp32 (the fused executors') and cross the wire as a bf16 copy; otherwise they are
        the wire format already (the module path: autograd accumulates into the buffer that is reduced)."""
        self.store, self.info, self.comm, self.stage_bf16 = store, info, comm, stage_bf16
        self.zero = zero and comm is None
        self.world = info.world_size
        self.transport = "none" if self.world == 1 else "p2p" if comm is not None else transport
        # the owned range of the optimizer state: 1/world under ZeRO-1 and in the peer-memory update (ZeRO-1 dataflow)
        if (self.zero or comm is not None) and self.world > 1:
            self.shard = store.shard_bounds(info.rank, self.world)
        else:
            self.shard = (0, store.numel)
        self._stage = None  # NCCL: the bf16 wire copy of fp32 gradients, allocated by the first update that needs it
        if comm is not None:
            # gradients travel as bf16 through a symmetric buffer, each rank updates its shard and writes the new parameters into
            # every replica
            self.param_buf = comm.buffer_of(store.params)
            self.grad_buf = comm.alloc(store.numel, torch.bfloat16) if stage_bf16 else comm.buffer_of(store.grads)
            self.gred = torch.empty(store.numel // self.world, dtype=torch.float32, device=store.device)

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
    def grad_norm_and_scale(self, max_norm: float, sumsq: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Return ``(total_norm, grad_scale)`` as device scalars.

        ``total_norm`` is the 2-norm of the world-averaged gradient (what ``clip_grad_norm_``
        reports upstream after DDP averaging); ``grad_scale = clip_coef / world``.  ``sumsq``: the sum of squares of the
        rank-summed gradient where the caller has it already, instead of the one taken here over the store's gradients.
        """
        sq = sumsq
        if sq is None:
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

    # ------------------------------------------------------------------ one optimizer update
    @torch.no_grad()
    def update(self, optimizer, clip: float, skip: Optional[torch.Tensor] = None, error_if_nonfinite: bool = False,
               local_loss: Optional[torch.Tensor] = None) -> UpdateInfo:
        """Reduce (once), norm and clip scale, AdamW, publish, zero the gradients: the update of every stepper on every transport."""
        if self.comm is not None:
            return self._peer_memory_update(optimizer, clip, skip, error_if_nonfinite, local_loss)
        grads = None
        if self.stage_bf16 and self.world > 1 and not self.zero:
            # NCCL baseline: gradients cross the wire as bf16 (like the reference's bf16 DDP buckets), once per update
            C = native.require()
            if self._stage is None:
                self._stage = torch.empty(self.store.numel, dtype=torch.bfloat16, device=self.store.device)
            grads = self._stage
            C.cast_f32_to_bf16(self.store.grads, grads, 1.0)
            dist.all_reduce(grads, op=dist.ReduceOp.SUM)
            sq = torch.zeros(1, dtype=torch.float32, device=self.store.device)
            C.sumsq(grads, sq)
            total, scale = self.grad_norm_and_scale(clip, sumsq=sq[0])
        else:
            self.reduce()
            total, scale = self.grad_norm_and_scale(clip)
        if error_if_nonfinite:
            _raise_if_nonfinite(total)
        optimizer.step(grad_scale=scale, skip=skip, grads=grads)
        self.gather_params()
        optimizer.zero_grad()
        return UpdateInfo(total)

    def _peer_memory_update(self, opt, clip, skip, error_if_nonfinite: bool, local_loss) -> UpdateInfo:
        """The data-parallel update on the hand-written NVLink kernels (``SymmComm.fused_update``): reduce-scatter + Σg² → norm /
        loss / skip exchange → AdamW on the owned shard → parameter broadcast.  ``skip`` and ``local_loss`` are this rank's values;
        a skip requested by any rank, or a non-finite gradient norm, leaves parameters, moments and the Adam step count untouched
        on every rank."""
        grp = opt.param_groups[0]
        dev = self.store.device
        sk = None if skip is None else (skip if torch.is_tensor(skip) else torch.tensor(float(skip), device=dev))
        opt.advance_step(None)  # optimistic: taken back below when the kernels skipped
        norm = self.comm.fused_update(
            grads_f32=self.store.grads if self.stage_bf16 else None, grad_buf=self.grad_buf, gred=self.gred, param_buf=self.param_buf,
            exp_avg=opt.exp_avg, exp_avg_sq=opt.exp_avg_sq,
            n=self.store.numel, lr=grp["lr"], betas=grp["betas"], eps=grp["eps"], weight_decay=grp["weight_decay"], step=opt.step_count,
            max_norm=clip, skip=sk, step_dev=opt._step_t, local_loss=local_loss)
        total = norm[0].clone()
        skip_count = self.comm.skip_all.clone()
        skipped_dev = (skip_count > 0).to(torch.float32)
        opt._step_t.sub_(skipped_dev)
        opt.undo_step_if_nonfinite(total, skipped_dev)
        opt.zero_grad()
        if error_if_nonfinite:
            _raise_if_nonfinite(total)
        mean_loss = self.comm.loss_out[0].clone() if local_loss is not None else None
        return UpdateInfo(total, mean_loss=mean_loss, skip_count=skip_count)


def _raise_if_nonfinite(total: torch.Tensor) -> None:
    """``clip_grad_norm_(error_if_nonfinite=True)`` of the reference loop (one host synchronisation)."""
    if not bool(torch.isfinite(total)):
        raise RuntimeError(f"The total norm of order 2.0 for gradients is non-finite ({float(total)}), so it cannot be clipped.")
