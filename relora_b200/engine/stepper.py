"""The per-update machinery shared by the trainer and ``bench.py``.

A *stepper* owns the model replica, the flat parameter store, the optimizer and the gradient
transport and exposes two calls:

    loss = stepper.micro_step(input_ids)      # forward + backward, gradients accumulate locally
    info = stepper.update(lr=None)            # reduce (once), clip, AdamW, zero grads

This mirrors one iteration of the reference hot loop (``torchrun_main.py:783-826``) with the
gradient all-reduce hoisted out of the accumulation loop.  :class:`ModuleStepper` drives any
``nn.Module`` whose forward returns ``.loss`` (CPU/gloo and the generic GPU path);
:class:`relora_b200.engine.fused_llama.FusedLlamaStepper` and
:class:`relora_b200.engine.fused_pythia.FusedPythiaStepper` are the H100 executors (whole-layer fused
kernels, CUDA graphs) with the same interface, built on :class:`relora_b200.engine.fused_common.FusedStepperBase`.
:func:`make_stepper` picks the executor: the module's ``supports`` / ``supports_full_rank`` decide, then
one constructor call builds it.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from ..parallel.dist import DistInfo
from ..parallel.flat import FlatAdamW, FlatParamStore
from ..parallel.grad_sync import GradSync, broadcast_params

__all__ = ["UpdateInfo", "ModuleStepper", "trainable_named_parameters", "make_stepper"]


@dataclass
class UpdateInfo:
    grad_norm: torch.Tensor  # device scalar (norm of the averaged gradient, before clipping)
    skipped: bool
    # set by the peer-memory update when the caller handed it this rank's loss: mean loss over ranks and the number of ranks that
    # asked to skip (device scalars; the reference's loss_info all-reduce folded into the kernel chain, torchrun_main.py:810)
    mean_loss: Optional[torch.Tensor] = None
    skip_count: Optional[torch.Tensor] = None


def trainable_named_parameters(model: torch.nn.Module) -> List[Tuple[str, torch.nn.Parameter]]:
    return [(n, p) for n, p in model.named_parameters() if p.requires_grad]


class ModuleStepper:
    def __init__(
        self,
        model: torch.nn.Module,
        info: DistInfo,
        *,
        lr: float,
        betas=(0.9, 0.999),
        eps: float = 1e-8,
        weight_decay: float = 0.0,
        clip_grad_norm: float = 1.0,
        grad_accumulation: int = 1,
        zero: bool = False,
        transport: str = "nccl",
        native=None,
    ):
        self.model, self.info = model, info
        self.ga = grad_accumulation
        self.clip = clip_grad_norm
        broadcast_params(model)
        named = trainable_named_parameters(model)
        # ---- transport: the hand-written NVLink update (csrc/comm.cu) when symmetric memory is available -- bf16 parameters on
        # CUDA, more than one rank -- and NCCL / gloo otherwise.  Same kernel chain as the fused executor, except that the bf16
        # gradients autograd accumulated are already in the symmetric buffer (no cast pass).
        self.comm = None
        p0 = named[0][1]
        if info.world_size > 1 and transport in ("p2p", "auto") and p0.is_cuda and p0.dtype == torch.bfloat16:
            from ..parallel.symm import SymmComm, symmetric_memory_available

            if symmetric_memory_available():
                try:
                    self.comm = SymmComm()
                except Exception as e:  # no P2P access, allocation failure, ...
                    if transport == "p2p":
                        raise
                    from ..obs import logger

                    logger.warning(f"peer-memory collectives unavailable ({type(e).__name__}: {e}); using NCCL")
            elif transport == "p2p":
                raise RuntimeError("--comm p2p needs torch symmetric memory over an NCCL process group")
        elif transport == "p2p" and info.world_size > 1:
            raise RuntimeError("--comm p2p needs bf16 parameters on CUDA")
        if self.comm is not None:
            alloc = self.comm.allocator()
            self.store = FlatParamStore(named, world_size=info.world_size, allocator=alloc, grad_allocator=alloc)
            self.sync = GradSync(self.store, info, transport="nccl", zero=False)
            self.sync.transport = "p2p"
            self.param_buf = self.comm.buffer_of(self.store.params)
            self.grad_buf = self.comm.buffer_of(self.store.grads)
            self.gred = torch.empty(self.store.numel // info.world_size, dtype=torch.float32, device=p0.device)
            shard = self.store.shard_bounds(info.rank, info.world_size)  # ZeRO-1 dataflow: each rank owns 1/world of the moments
        else:
            self.store = FlatParamStore(named, world_size=info.world_size)
            self.sync = GradSync(self.store, info, transport="nccl", zero=zero)
            shard = self.sync.shard if zero else None
        self.optimizer = FlatAdamW(self.store, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                   shard=shard, native=native)
        self.trainable_params = [p for _, p in named]
        self.trainable_names = [n for n, _ in named]
        self.lora_params = [p for n, p in named if "lora_" in n]

    # ------------------------------------------------------------------ one micro-batch
    def micro_step(self, input_ids: torch.Tensor) -> torch.Tensor:
        out = self.model(input_ids=input_ids, labels=input_ids)
        loss = out.loss
        (loss / self.ga).backward()
        if input_ids.is_cuda:  # fresh LoRA-dropout masks for the next micro-batch (device-side counter)
            from ..ops import fused

            fused.seed_state.advance(input_ids.device)
        return loss.detach()

    @torch.no_grad()
    def eval_loss(self, input_ids: torch.Tensor) -> torch.Tensor:
        return self.model(input_ids=input_ids, labels=input_ids).loss.detach()

    # ------------------------------------------------------------------ one optimizer update
    @property
    def folds_loss_reduce(self) -> bool:
        """True when ``update(local_loss=...)`` combines loss / skip over ranks inside the NVLink kernel chain (no NCCL call)."""
        return self.comm is not None

    @torch.no_grad()
    def update(self, skip: Optional[torch.Tensor] = None, error_if_nonfinite: bool = False,
               local_loss: Optional[torch.Tensor] = None) -> UpdateInfo:
        if self.comm is not None:
            return peer_memory_update(self, grads_f32=None, skip=skip, error_if_nonfinite=error_if_nonfinite, local_loss=local_loss)
        self.sync.reduce()
        total, scale = self.sync.grad_norm_and_scale(self.clip)
        if error_if_nonfinite and not bool(torch.isfinite(total)):
            raise RuntimeError(
                f"The total norm of order 2.0 for gradients is non-finite ({float(total)}), so it cannot be clipped."
            )
        skipped = bool(skip) if skip is not None and not self.store.params.is_cuda else False
        self.optimizer.step(grad_scale=scale, skip=skip)
        self.sync.gather_params()
        self.optimizer.zero_grad()
        return UpdateInfo(total, skipped)

    def set_lr(self, lr: float) -> None:
        for g in self.optimizer.param_groups:
            g["lr"] = lr


def peer_memory_update(st, *, grads_f32, skip, error_if_nonfinite: bool, local_loss) -> UpdateInfo:
    """The data-parallel update on the hand-written NVLink kernels (``SymmComm.fused_update``), shared by both steppers: reduce-
    scatter + Σg² → norm / loss / skip exchange → AdamW on the owned shard → parameter broadcast.  ``skip`` and ``local_loss`` are
    this rank's values; a skip requested by any rank, or a non-finite gradient norm, leaves parameters, moments and the Adam step
    count untouched on every rank."""
    opt = st.optimizer
    grp = opt.param_groups[0]
    dev = st.store.device
    sk = None if skip is None else (skip if torch.is_tensor(skip) else torch.tensor(float(skip), device=dev))
    opt.advance_step(None)  # optimistic: taken back below when the kernels skipped
    norm = st.comm.fused_update(
        grads_f32=grads_f32, grad_buf=st.grad_buf, gred=st.gred, param_buf=st.param_buf, exp_avg=opt.exp_avg, exp_avg_sq=opt.exp_avg_sq,
        n=st.store.numel, lr=grp["lr"], betas=grp["betas"], eps=grp["eps"], weight_decay=grp["weight_decay"], step=opt.step_count,
        max_norm=st.clip, skip=sk, step_dev=opt._step_t, local_loss=local_loss)
    total = norm[0].clone()
    skip_count = st.comm.skip_all.clone()
    skipped_dev = (skip_count > 0).to(torch.float32)
    opt._step_t.sub_(skipped_dev)
    opt.undo_step_if_nonfinite(total, skipped_dev)
    opt.zero_grad()
    if error_if_nonfinite and not bool(torch.isfinite(total)):
        raise RuntimeError(f"The total norm of order 2.0 for gradients is non-finite ({float(total)}), so it cannot be clipped.")
    mean_loss = st.comm.loss_out[0].clone() if local_loss is not None else None
    return UpdateInfo(total, False, mean_loss=mean_loss, skip_count=skip_count)


def make_stepper(model, info: DistInfo, args, *, native=None):
    """Pick the executor for ``model`` on ``info.device`` according to ``--engine``."""
    engine = getattr(args, "engine", "auto")
    zero = str(args.optimizer).lower() == "adam_zero"
    transport = getattr(args, "comm", "auto")
    kw = dict(
        lr=args.lr,
        betas=(args.adam_beta1, args.adam_beta2),
        weight_decay=args.weight_decay,
        clip_grad_norm=args.clip_grad_norm,
        grad_accumulation=args.gradient_accumulation,
        zero=zero,
        transport=transport,
        native=native,
    )
    if engine in ("auto", "fused") and info.device.type == "cuda":
        from ..models.llama import LlamaForCausalLM
        from ..models.pythia import GPTNeoXForCausalLM
        from . import fused_llama, fused_pythia

        frozen = getattr(args, "frozen_dtype", None)
        ok, why = fused_llama.supports(model, args)
        cls = fused_llama.FusedLlamaStepper if ok else None
        if cls is None and engine == "fused":
            # Pythia (GPT-NeoX) and full-rank Llama run fused only on request; `auto` keeps both on the module path
            inner = getattr(model, "wrapped_model", model)
            if isinstance(model, LlamaForCausalLM):
                cls, check = fused_llama.FusedLlamaStepper, fused_llama.supports_full_rank
            elif isinstance(model, GPTNeoXForCausalLM):
                cls, check = fused_pythia.FusedPythiaStepper, fused_pythia.supports_full_rank
            else:
                cls, check = fused_pythia.FusedPythiaStepper, fused_pythia.supports
            ok, why_fused = check(model, args)
            if not ok:
                # a wrapped model that is not GPT-NeoX keeps the Llama executor's reason
                keep_llama_why = check is fused_pythia.supports and not isinstance(inner, GPTNeoXForCausalLM)
                raise RuntimeError(f"--engine fused requested but not applicable: {why if keep_llama_why else why_fused}")
        if cls is not None:
            if cls is fused_llama.FusedLlamaStepper:
                kw.update(fp8=frozen in ("fp8", "fp8_full"), fp8_backward=frozen == "fp8_full")
            return cls(model, info, cuda_graphs=getattr(args, "cuda_graphs", True), attention=getattr(args, "attention", "auto"),
                       deterministic=bool(getattr(args, "deterministic", False)), **kw)
    if info.device.type != "cuda":
        kw["transport"] = "nccl"  # CPU: the process group's own reduction (gloo)
    # the fp8 tensor-core path and the wgmma attention kernels belong to the fused executor: say so instead of silently
    # training in bf16 / with SDPA
    from ..obs import logger

    if getattr(args, "frozen_dtype", None) in ("fp8", "fp8_full"):
        logger.warning(f"--frozen_dtype {args.frozen_dtype} needs the fused executor (Llama + ReLoRA on CUDA/bf16); "
                       "the module path runs the frozen weights in the model dtype")
    if getattr(args, "attention", "auto") in ("sdpa", "native"):
        import os as _os

        _os.environ["RELORA_B200_ATTENTION"] = args.attention  # the module path reads the switch where it calls attention
    return ModuleStepper(model, info, **kw)
