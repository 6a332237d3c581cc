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

from typing import List, Optional, Tuple

import torch

from ..parallel.dist import DistInfo
from ..parallel.flat import FlatAdamW, FlatParamStore
from ..parallel.grad_sync import GradSync, UpdateInfo, broadcast_params, peer_transport
from ..relora import ReLoRaModel, get_scheduler, optimizer_reset

__all__ = ["UpdateInfo", "Stepper", "ModuleStepper", "trainable_named_parameters", "make_stepper", "wrap_relora", "make_scheduler",
           "reset_optimizer"]


def trainable_named_parameters(model: torch.nn.Module) -> List[Tuple[str, torch.nn.Parameter]]:
    return [(n, p) for n, p in model.named_parameters() if p.requires_grad]


class Stepper:
    """What every stepper has.  A subclass sets ``model``, ``info`` and ``clip``, picks ``comm`` (:func:`peer_transport`), carves
    ``store`` out of that transport's allocator -- the symmetric allocation has to exist first -- and then calls ``_init_update``;
    ``micro_step`` and ``eval_loss`` are its own."""

    def _init_update(self, *, zero: bool, stage_bf16: bool, native, **adamw) -> None:
        self.sync = GradSync(self.store, self.info, zero=zero, comm=self.comm, stage_bf16=stage_bf16)
        self.optimizer = FlatAdamW(self.store, shard=self.sync.shard, native=native, **adamw)
        self.trainable_params, self.trainable_names = list(self.store.param_list), list(self.store.names)
        self.lora_params = [p for n, p in zip(self.trainable_names, self.trainable_params) if "lora_" in n]

    @property
    def folds_loss_reduce(self) -> bool:
        """True when ``update(local_loss=...)`` combines loss / skip over ranks inside the NVLink kernel chain (no NCCL call)."""
        return self.comm is not None

    def update(self, skip: Optional[torch.Tensor] = None, error_if_nonfinite: bool = False,
               local_loss: Optional[torch.Tensor] = None) -> UpdateInfo:
        return self.sync.update(self.optimizer, self.clip, skip, error_if_nonfinite, local_loss)

    def set_lr(self, lr: float) -> None:
        for g in self.optimizer.param_groups:
            g["lr"] = lr

    def merge_and_reinit(self) -> None:
        self.model.merge_and_reinit()


class ModuleStepper(Stepper):
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
        # the hand-written NVLink update needs bf16 parameters on CUDA.  Same kernel chain as the fused executor, except that the
        # bf16 gradients autograd accumulated are already in the symmetric buffer (no cast pass).
        p0 = named[0][1]
        self.comm = peer_transport(info, transport, eligible=p0.is_cuda and p0.dtype == torch.bfloat16)
        alloc = self.comm.allocator() if self.comm is not None else None
        self.store = FlatParamStore(named, world_size=info.world_size, allocator=alloc, grad_allocator=alloc)
        self._init_update(zero=zero, stage_bf16=False, native=native, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)

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


def wrap_relora(model: torch.nn.Module, args, *, lora_only: bool) -> ReLoRaModel:
    """``model`` under ReLoRA as the command line describes it."""
    model = ReLoRaModel(
        model, r=args.lora_r, lora_alpha=args.lora_alpha, lora_dropout=args.lora_dropout,
        target_modules=["attn", "attention", "mlp"], trainable_scaling=args.train_scaling,
        keep_original_weights=True, lora_only=lora_only, quantize=args.quantize,
        use_double_quant=args.use_double_quant, init_lora_a=args.init_lora_a,
    )
    model.seed = args.seed
    return model


def make_scheduler(optimizer, args, num_training_steps: int):
    return get_scheduler(
        optimizer, scheduler_type=args.scheduler, num_training_steps=num_training_steps,
        warmup_steps=args.warmup_steps, min_lr_ratio=args.min_lr_ratio, cycle_length=args.cycle_length,
        restart_warmup_steps=args.restart_warmup_steps, adjust_step=args.adjust_step,
    )


def reset_optimizer(optimizer, lora_params, args, reset_index: int) -> float:
    """Prune the Adam moments of the LoRA factors (the ``reset_index``-th reset of the run keys the random pruning)."""
    return optimizer_reset(
        optimizer, reset_params=lora_params, optimizer_state_keys=["exp_avg", "exp_avg_sq"],
        reset_optimizer_on_relora=args.reset_optimizer_on_relora, optimizer_random_pruning=args.optimizer_random_pruning,
        optimizer_magnitude_pruning=args.optimizer_magnitude_pruning, seed=args.seed, reset_index=reset_index,
    )


def make_stepper(model, info: DistInfo, args, *, native=None, dropout_seed: Optional[int] = None):
    """Pick the executor for ``model`` on ``info.device`` according to ``--engine``.  On CUDA the optimizer runs on the extension's
    AdamW (``native``, created here unless given) and the LoRA-dropout counter starts from ``dropout_seed`` (a resumed run's saved
    counter) or, without one, from a value derived from ``--seed``, so runs with different seeds draw different masks.
    ``--activation_checkpointing`` turns on the models' per-layer ``torch.utils.checkpoint`` and the fused executors' recompute."""
    checkpointing = bool(getattr(args, "activation_checkpointing", False))
    if checkpointing:
        getattr(model, "wrapped_model", model).gradient_checkpointing_enable()
    if info.device.type == "cuda":
        from ..ops import fused, reference
        from ..ops import native as extension

        extension.require()  # a CUDA device without the sm_90a extension fails here, before any training step
        native = native or fused.NativeOptim()
        if dropout_seed is None and hasattr(args, "seed"):  # a hand-made namespace without --seed leaves the counter alone
            dropout_seed = reference.mix_seed(args.seed, 0x5eed)
        if dropout_seed is not None:
            fused.seed_state.set(info.device, dropout_seed)
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
        quantized = isinstance(model, ReLoRaModel) and model._config.quantize is not None
        if cls is None and engine == "fused" and quantized:
            # MXFP8-packed frozen weights run fused only on request; `auto` keeps quantised models on the module path
            exe = fused_pythia if isinstance(model.wrapped_model, GPTNeoXForCausalLM) else fused_llama
            ok, why_q = exe.supports_quantized(model, args)
            if not ok:
                raise RuntimeError(f"--engine fused requested but not applicable: {why_q}")
            cls = fused_pythia.FusedPythiaStepper if exe is fused_pythia else fused_llama.FusedLlamaStepper
            kw["quantize"] = "mxfp8"
        elif cls is None and engine == "fused":
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
            if cls is fused_llama.FusedLlamaStepper and "quantize" not in kw:
                kw.update(fp8=frozen in ("fp8", "fp8_full"), fp8_backward=frozen == "fp8_full")
            if checkpointing:
                kw["activation_checkpointing"] = True
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
