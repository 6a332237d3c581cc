"""NVLink peer-memory communication: symmetric buffers + the hand-written collectives of ``csrc/comm.cu``.

``SymmComm`` owns the cross-rank bookkeeping (flag area, epochs); ``SymmBuffer`` is one allocation that every
rank can address directly (``torch.distributed._symmetric_memory``: CUDA VMM allocation, handles exchanged over
the process group's store, optional NVLS multicast alias).  Kernels:

* ``all_reduce_``   — two-shot in-place all-reduce of a bf16 range (reduce-scatter by the owner of each chunk with
  fp32 accumulation, result stored straight into every peer); with a multicast mapping the reduction happens in
  the NVSwitch (``multimem.ld_reduce``) and the result is broadcast with ``multimem.st``;
* ``fused_update``  — the whole data-parallel optimizer update as one kernel chain:
  bf16 cast → reduce-scatter + Σg² → norm exchange / clip coefficient → AdamW on the owned shard →
  parameter broadcast into every replica (ZeRO-1 dataflow; bit-identical parameters on all ranks).

NCCL (``GradSync(transport="nccl")``) remains the baseline and the fallback when symmetric memory is unavailable.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

from ..obs import logger
from ..ops import native

__all__ = ["SymmComm", "SymmBuffer", "symmetric_memory_available"]


def symmetric_memory_available() -> bool:
    if not (dist.is_initialized() and torch.cuda.is_available() and dist.get_backend() == "nccl"):
        return False
    try:
        import importlib

        importlib.import_module("torch.distributed._symmetric_memory")
        return True
    except Exception:
        return False


class SymmBuffer:
    """A tensor allocated in symmetric memory plus the peers' views of it."""

    def __init__(self, tensor: torch.Tensor, handle):
        self.tensor = tensor
        self.handle = handle
        # the tensor may start at a byte offset inside the allocation (torch sub-allocates symmetric memory from a pool in some
        # configurations): every peer view and the multicast alias are shifted by it, so ptrs[rank] == tensor.data_ptr()
        off = int(getattr(handle, "offset", 0) or 0)
        self.base_offset = off
        self.ptrs: List[int] = [int(p) + off for p in handle.buffer_ptrs]
        mc = 0
        try:
            if handle.has_multicast_support:
                mc = int(handle.multicast_ptr) + off
        except Exception:
            mc = 0
        self.mc_base = mc
        rank = int(getattr(handle, "rank", -1))
        if 0 <= rank < len(self.ptrs) and self.ptrs[rank] != tensor.data_ptr():
            raise RuntimeError(f"symmetric buffer: local peer view {self.ptrs[rank]:#x} does not alias the tensor ({tensor.data_ptr():#x}, "
                               f"offset {off})")

    def mc_ptr(self, use_multicast: bool) -> int:
        return self.mc_base if (use_multicast and self.mc_base) else 0


class SymmComm:
    def __init__(self, group=None, use_multicast: Optional[bool] = None, max_blocks: int = 128):
        import torch.distributed._symmetric_memory as symm_mem

        self._symm = symm_mem
        self.group = group or dist.group.WORLD
        self.rank = dist.get_rank(self.group)
        self.world = dist.get_world_size(self.group)
        if self.world > 8:
            raise RuntimeError("the peer-memory collectives address at most 8 GPUs (one NVSwitch domain)")
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.C = native.require()
        if use_multicast is None:
            # NVLS (multimem.ld_reduce / multimem.st through the switch) above 4 ranks, plain peer loads / stores below; this crossover
            # has not been measured on H100 boxes (bench/allreduce_bench.py measures both)
            env = os.environ.get("RELORA_B200_MULTICAST")
            use_multicast = (env == "1") if env is not None else self.world > 4
        self.use_multicast = use_multicast
        self.max_blocks = max_blocks
        self.epoch = 0
        flags = self.alloc(128, torch.int32)
        flags.tensor.zero_()
        self.flags = flags
        self.local_go = torch.zeros(2, dtype=torch.int32, device=self.device)
        self.scratch = torch.zeros(4, dtype=torch.float32, device=self.device)  # sum(g^2), grad scale, combined skip flag
        self.loss_out = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.norm_out = torch.zeros(1, dtype=torch.float32, device=self.device)
        torch.cuda.synchronize()
        dist.barrier(self.group)

    # ------------------------------------------------------------------ allocation
    def alloc(self, numel: int, dtype: torch.dtype) -> SymmBuffer:
        t = self._symm.empty(numel, dtype=dtype, device=self.device)
        h = self._symm.rendezvous(t, self.group)
        return SymmBuffer(t, h)

    def allocator(self):
        """``allocator(numel, dtype, device) -> tensor`` for :class:`FlatParamStore` (remembers the SymmBuffers)."""
        self._allocated = getattr(self, "_allocated", {})

        def _alloc(n, dt, dev):
            buf = self.alloc(n, dt)
            buf.tensor.zero_()
            self._allocated[buf.tensor.data_ptr()] = buf
            return buf.tensor

        return _alloc

    def buffer_of(self, tensor: torch.Tensor) -> Optional[SymmBuffer]:
        return getattr(self, "_allocated", {}).get(tensor.data_ptr())

    def _next_epoch(self) -> int:
        self.epoch += 1
        return self.epoch

    # ------------------------------------------------------------------ collectives
    def barrier(self) -> None:
        self.C.comm_barrier(self.flags.ptrs, self.rank, self.world, self.local_go, 3, self._next_epoch())

    def all_reduce_(self, buf: SymmBuffer, off_elems: int = 0, n: Optional[int] = None) -> None:
        """In-place sum over ranks of ``buf.tensor[off : off+n]`` (bf16)."""
        assert buf.tensor.dtype == torch.bfloat16
        n = buf.tensor.numel() - off_elems if n is None else n
        self.C.comm_allreduce_bf16(self.flags.ptrs, self.rank, self.world, self.local_go, buf.ptrs, buf.mc_ptr(self.use_multicast),
                                   off_elems, n, self._next_epoch(), self.max_blocks)

    def fused_update(self, *, grads_f32: Optional[torch.Tensor], grad_buf: SymmBuffer, gred: torch.Tensor, param_buf: SymmBuffer,
                     exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, n: int, lr: float, betas: Tuple[float, float], eps: float,
                     weight_decay: float, step: int, max_norm: float, skip: Optional[torch.Tensor],
                     step_dev: Optional[torch.Tensor] = None, local_loss: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Returns the gradient norm (device).  ``skip`` / ``local_loss`` are this rank's values: the kernel chain combines them over
        ranks (``self.skip_all``: number of ranks that asked to skip, ``self.loss_out``: mean loss) without an NCCL call."""
        sk = None if skip is None else skip.reshape(1).float()
        ll = None if local_loss is None else local_loss.reshape(1).float()
        self.C.comm_fused_update(self.flags.ptrs, self.rank, self.world, self.local_go, grads_f32, grad_buf.ptrs,
                                 grad_buf.mc_ptr(self.use_multicast), gred, param_buf.ptrs, param_buf.mc_ptr(self.use_multicast),
                                 exp_avg, exp_avg_sq, n, float(lr), float(betas[0]), float(betas[1]), float(eps), float(weight_decay),
                                 int(step), float(max_norm), sk, self.norm_out, self.scratch, self._next_epoch(), self.max_blocks,
                                 None if step_dev is None else step_dev.reshape(1).float(), ll, self.loss_out if ll is not None else None)
        return self.norm_out

    @property
    def skip_all(self) -> torch.Tensor:
        """Device scalar written by the last fused_update: how many ranks requested a skip (0 = the update was applied)."""
        return self.scratch[2]
