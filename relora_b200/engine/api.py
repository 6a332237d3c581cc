"""Programmatic front door: build a ready-to-train ReLoRA engine and drive it step by step.

    eng = TrainingEngine.build(model_config="configs/llama_250m.json", batch_size=24,
                               gradient_accumulation=6, max_length=512, use_peft=True, relora=5000, ...)
    loss = eng.train_step(batch)      # batch: pinned CPU int64 [ga, B, T]; H2D copy, ga micro-steps,
                                      # one optimizer update, LR schedule, ReLoRA resets; returns float

This is the call a library user (and ``bench.py``'s end-to-end measurement) makes; the CLI trainer
(:func:`relora_b200.engine.trainer.run`) wraps the same pieces with data loading and checkpointing.
"""
from __future__ import annotations

import argparse
from typing import Optional

import torch
import torch.distributed as dist

from ..config import build_parser, check_args
from ..models import LlamaForCausalLM, load_config
from ..parallel.dist import DistInfo, init_distributed
from .stepper import make_scheduler, make_stepper, reset_optimizer, wrap_relora

__all__ = ["TrainingEngine"]


class TrainingEngine:
    def __init__(self, args: argparse.Namespace, info: Optional[DistInfo] = None):
        self.args = args
        self.info = info or init_distributed(args.device, args.backend)
        device = self.info.device
        torch.manual_seed(args.seed)
        cfg = load_config(args.model_config)
        model = LlamaForCausalLM(cfg)
        if args.use_peft:
            model = wrap_relora(model, args, lora_only=False)
        dtype = torch.bfloat16 if args.dtype in ("bf16", "bfloat16") else torch.float32
        self.model = model.to(device=device, dtype=dtype)
        self.model.train()
        self.stepper = make_stepper(self.model, self.info, args)
        self.optimizer = self.stepper.optimizer
        self.scheduler = make_scheduler(self.optimizer, args, args.num_training_steps)
        self.update_step = 0
        self.n_lora_restarts = 0
        self.n_optimizer_resets = 0
        self._nan = torch.zeros((), dtype=torch.float32, device=device)
        self._dev_batch = None
        self._loss_host = torch.zeros(1, dtype=torch.float32).pin_memory() if device.type == "cuda" else torch.zeros(1)

    # ------------------------------------------------------------------ construction helpers
    @classmethod
    def build(cls, info: Optional[DistInfo] = None, **overrides) -> "TrainingEngine":
        """Keyword arguments are the CLI flags of ``torchrun_main.py`` (``lr=1e-3``, ``relora=5000`` …)."""
        parser = build_parser()
        args = parser.parse_args([])
        for k, v in overrides.items():
            if not hasattr(args, k):
                raise TypeError(f"unknown option {k!r}")
            setattr(args, k, v)
        if args.synthetic_data is None and args.dataset_path is None and args.megatron_dataset_config is None:
            args.synthetic_data = "0"  # data is supplied by the caller, step by step
        args = check_args(args, argv=[])
        world = int(dist.get_world_size()) if dist.is_initialized() else int(__import__("os").environ.get("WORLD_SIZE", "1"))
        if args.gradient_accumulation is None:
            args.gradient_accumulation = max(1, args.total_batch_size // (args.batch_size * world))
        return cls(args, info)

    # ------------------------------------------------------------------ stepping
    def train_step_device(self, ids: torch.Tensor) -> torch.Tensor:
        """One optimizer update from device-resident token ids ``[ga, B, T]``; returns the mean loss
        of the micro-batches as a device scalar (no host synchronisation)."""
        a = self.args
        ga = ids.shape[0]
        total = None
        for i in range(ga):
            loss = self.stepper.micro_step(ids[i])
            total = loss.float() if total is None else total + loss.float()
        mean = total / ga
        self.last_local_loss = mean  # this rank's loss before the cross-rank mean (device scalar; bench.py's validity check)
        skip = torch.isnan(mean).float()
        multi = dist.is_initialized() and dist.get_world_size() > 1
        if multi and getattr(self.stepper, "folds_loss_reduce", False):
            # the NVLink update combines [loss, NaN flag] over ranks in its norm exchange: no NCCL call on the step path
            info = self.stepper.update(skip=skip, local_loss=mean)
            mean = info.mean_loss
        else:
            if multi:
                pack = torch.stack([mean, skip])
                dist.all_reduce(pack)
                mean, skip = pack[0] / dist.get_world_size(), pack[1]
            info = self.stepper.update(skip=skip)
        self.last_grad_norm = info.grad_norm
        # the fused / flat optimizers step inside update(); mark the wrapped torch counter so LambdaLR does not warn about order
        self.optimizer._opt_called = True
        self.scheduler.step()
        self.update_step += 1
        self._maybe_reset()
        return mean

    def train_step(self, batch: torch.Tensor) -> float:
        """End-to-end step: pinned-host ``batch`` → device, update, loss back to the host."""
        dev = self.info.device
        if dev.type == "cuda":
            if self._dev_batch is None or self._dev_batch.shape != batch.shape:
                self._dev_batch = torch.empty(batch.shape, dtype=batch.dtype, device=dev)
            self._dev_batch.copy_(batch, non_blocking=True)
            loss = self.train_step_device(self._dev_batch)
            self._loss_host.copy_(loss.reshape(1), non_blocking=True)
            torch.cuda.current_stream().synchronize()
            return float(self._loss_host[0])
        return float(self.train_step_device(batch.to(dev)))

    def _maybe_reset(self):
        a = self.args
        if a.relora is None:
            return
        if self.update_step >= a.relora and self.update_step % a.relora == 1:
            self.n_lora_restarts += 1
            self.stepper.merge_and_reinit()
        if self.update_step >= a.cycle_length and self.update_step % a.cycle_length == 1:
            self.n_optimizer_resets += 1
            reset_optimizer(self.optimizer, self.stepper.lora_params, a, self.n_optimizer_resets)

    @property
    def tokens_per_step(self) -> int:
        a = self.args
        return a.batch_size * a.gradient_accumulation * a.max_length * self.info.world_size
