"""Command-line / YAML configuration of the trainer.

Same flag surface and post-processing as the reference (``torchrun_main.py:54-140`` and
``peft_pretraining/args_utils.py:8-86``), with these deliberate fixes:

* boolean flags accept both ``--use_peft`` and ``--use_peft true|false`` (upstream requires a value,
  which breaks its own README examples);
* ``cycle_length`` defaults to ``relora`` when a ReLoRA run does not set it (the shipped
  ``1B_v1.0.yaml`` omits it and would crash upstream);
* ``--training_config`` may be combined with engine flags (``--device``, ``--comm`` ...), but not
  with training hyper-parameters, which stay an error like upstream.

Engine-only flags (no upstream equivalent) are grouped at the bottom of :func:`build_parser`.
"""
from __future__ import annotations

import argparse
import os
import sys
from typing import List, Optional

import yaml

from .obs import logger

__all__ = ["build_parser", "parse_args", "check_args", "max_train_tokens_to_number", "ENGINE_FLAGS"]


def max_train_tokens_to_number(s) -> int:
    """``"100M"`` → 100_000_000, ``"1B"`` → 1_000_000_000 (reference training_utils.py:239-245)."""
    if isinstance(s, int):
        return s
    s = str(s)
    if s.endswith("M"):
        return int(s[:-1]) * 1_000_000
    if s.endswith("B"):
        return int(s[:-1]) * 1_000_000_000
    return int(s)


def _bool(v) -> bool:
    if isinstance(v, bool):
        return v
    return str(v).lower() == "true"


def _add_bool(parser, name: str, default: bool, help: Optional[str] = None):
    parser.add_argument(name, default=default, type=_bool, nargs="?", const=True, help=help)


def _default_dtype() -> str:
    try:
        import torch

        if torch.cuda.is_available() and not torch.cuda.is_bf16_supported():
            return "float32"
    except Exception:  # pragma: no cover
        pass
    return "bfloat16"


# flags that only exist in this engine; allowed next to --training_config
ENGINE_FLAGS = (
    "--device", "--backend", "--comm", "--engine", "--lora_dropout", "--cuda_graphs", "--frozen_dtype",
    "--init_lora_a", "--synthetic_data", "--log_every", "--parity_quirks", "--attention", "--deterministic",
    "--activation_checkpointing",
)


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="ReLoRA pre-training (H100-native engine)")
    p.add_argument("--training_config", type=str, default=None,
                   help="Path to a yaml file with the training run config; overrides all parameters.")

    p.add_argument("--model_config", type=str, default=None)
    p.add_argument("--model_name_or_path", type=str, default=None, help="Local HF checkpoint directory (Pythia), alternative to --model_config")
    p.add_argument("--model_revision", type=str, default=None)
    p.add_argument("--warmed_up_model", type=str, default=None, help="Start from warmed-up weights; optimizer/scheduler are not restored.")
    p.add_argument("--resume_from", type=str, default=None, help="Continue training, loading optimizer and scheduler from the checkpoint.")
    _add_bool(p, "--load_optimizer_state_on_resume", True)

    p.add_argument("--dataset_path", type=str, default=None, help="Path to a pre-tokenized HF dataset directory")
    p.add_argument("--megatron_dataset_config", type=str, default=None, help="Path to a Megatron/NeoX dataset yaml")
    p.add_argument("--max_length", type=int, default=512)

    p.add_argument("--batch_size", type=int, default=None)
    p.add_argument("--gradient_accumulation", type=int, default=None)
    p.add_argument("--total_batch_size", type=int, default=None)

    _add_bool(p, "--use_peft", False)
    p.add_argument("--lora_r", type=int, default=128)
    p.add_argument("--lora_alpha", type=float, default=32)
    p.add_argument("--relora", type=int, default=None)
    p.add_argument("--train_scaling", default=False, action="store_true")
    _add_bool(p, "--reset_optimizer_on_relora", True)
    p.add_argument("--optimizer_random_pruning", default=0.0, type=float)
    p.add_argument("--optimizer_magnitude_pruning", default=0.0, type=float)
    _add_bool(p, "--force_keep_original", False)

    p.add_argument("--optimizer", default="Adam", help="adam (AdamW) or adam_zero (optimizer-state sharding)")
    p.add_argument("--lr", type=float, default=1e-4)
    p.add_argument("--scheduler", type=str, default="cosine", choices=["linear", "cosine", "cosine_restarts"])
    p.add_argument("--cycle_length", type=int, default=None)
    p.add_argument("--restart_warmup_steps", type=int, default=None)
    p.add_argument("--adjust_step", type=int, default=0)
    p.add_argument("--min_lr_ratio", type=float, default=0.1)
    p.add_argument("--adam_beta1", type=float, default=0.9)
    p.add_argument("--adam_beta2", type=float, default=0.999)
    p.add_argument("--weight_decay", type=float, default=0.0)
    p.add_argument("--warmup_steps", type=int, default=1_000)
    p.add_argument("--clip_grad_norm", type=float, default=1.0)

    p.add_argument("--eval_every", type=int, default=1_000)
    p.add_argument("--num_training_steps", type=int, default=10_000, help="Number of update steps.")
    p.add_argument("--max_train_tokens", type=max_train_tokens_to_number, default=None)
    p.add_argument("--save_every", type=int, default=10_000)
    p.add_argument("--save_dir", type=str, default=None)
    p.add_argument("--keep_checkpoints", type=int, default=None)
    p.add_argument("--tags", type=str, default=None)
    p.add_argument("--dtype", type=str, default=_default_dtype())
    p.add_argument("--workers", type=int, default=8)

    p.add_argument("--quantize", default=None, type=str, choices=[None, "4bit", "8bit", "nvfp4", "mxfp8", "fp4", "fp8"])
    _add_bool(p, "--use_double_quant", True)

    p.add_argument("--distributed_type", type=str, default="ddp", choices=["fsdp", "ddp"])
    _add_bool(p, "--profile", False)
    _add_bool(p, "--autoresume", False)
    p.add_argument("--comment", type=str, default=None)
    _add_bool(p, "--wandb_watch", False)
    p.add_argument("--skip_batches", default=None, type=str, help="Update-step numbers to skip, comma separated.")
    p.add_argument("--seed", type=int, default=0)

    # ---- engine flags (this repository only) ----
    p.add_argument("--device", type=str, default="auto", choices=["auto", "cuda", "cpu"])
    p.add_argument("--backend", type=str, default="auto", choices=["auto", "nccl", "gloo"])
    p.add_argument("--comm", type=str, default="auto", choices=["auto", "nccl", "p2p"],
                   help="gradient all-reduce: NCCL baseline or the NVLink peer-memory kernels")
    p.add_argument("--engine", type=str, default="auto", choices=["auto", "fused", "module"],
                   help="fused: whole-layer sm_90a executor (+CUDA graphs); module: nn.Module path")
    p.add_argument("--lora_dropout", type=float, default=0.1, help="hard-coded to 0.1 upstream (torchrun_main.py:546)")
    _add_bool(p, "--cuda_graphs", True)
    _add_bool(p, "--deterministic", False,
              help="fixed summation order for the weight-gradient GEMMs (no split-K atomics; slower) on top of the always-deterministic embedding backward")
    p.add_argument("--attention", type=str, default="auto", choices=["auto", "native", "sdpa"],
                   help="native: wgmma flash-attention kernels of this repo (head_dim a multiple of 8, <= 256); sdpa: torch SDPA (cuDNN); "
                        "auto: the kernels for head_dim <= 64, SDPA above")
    p.add_argument("--frozen_dtype", type=str, default=None, choices=[None, "bf16", "fp8", "fp8_full", "mxfp8", "nvfp4"],
                   help="fp8: E4M3 tensor-core path for the frozen weights on the fused executor (per-tensor scales, delayed "
                        "activation scaling), forward GEMMs only; fp8_full: also the input-gradient GEMMs (E5M2 gradients); mxfp8 / nvfp4: block-scaled storage on the module path (alias of --quantize)")
    p.add_argument("--init_lora_a", type=str, default="zeros", choices=["zeros", "kaiming"],
                   help="zeros reproduces upstream (both LoRA factors zero until the first reset)")
    p.add_argument("--synthetic_data", type=str, default=None,
                   help="'<n_sequences>' — train on random token ids instead of a dataset on disk")
    p.add_argument("--log_every", type=int, default=1)
    _add_bool(p, "--activation_checkpointing", False,
              help="keep only each layer's input (and the wgmma attention's output) for the backward and recompute the rest of the "
                   "layer there: about one more forward of the projections per step for activation memory that no longer grows "
                   "with the number of layers")
    _add_bool(p, "--parity_quirks", True, help="keep upstream quirks (dataset-size check units, token/sequence step math)")
    return p


def _cli_has_training_flags(argv: List[str]) -> bool:
    flags = [a for a in argv if a.startswith("--")]
    extra = [f for f in flags if f.split("=")[0] not in ("--training_config",) + ENGINE_FLAGS]
    return len(extra) > 0


def check_args(args: argparse.Namespace, argv: Optional[List[str]] = None) -> argparse.Namespace:
    """Post-process and validate (reference ``args_utils.check_args_torchrun_main``)."""
    if args.training_config is not None:
        logger.info(f"Yaml config provided for the run. The file {args.training_config} is used to provide all the parameters.")
        if _cli_has_training_flags(sys.argv[1:] if argv is None else argv):
            raise RuntimeError(
                "You provided both a yaml config and command line arguments. "
                "Please use only one of the two options."
            )
        with open(args.training_config) as f:
            cfg = yaml.safe_load(f)
        for k, v in cfg.items():
            if k == "lr":
                v = float(v)
            if k == "max_train_tokens" and v is not None:
                v = max_train_tokens_to_number(v)
            setattr(args, k, v)

    if args.synthetic_data is None and (args.dataset_path is None) == (args.megatron_dataset_config is None):
        raise ValueError(
            "Either --dataset_path or --megatron_dataset_config must be specified and not both\n"
            f"Got {args.dataset_path=} and {args.megatron_dataset_config=}"
        )
    if args.megatron_dataset_config is not None and not os.path.exists(args.megatron_dataset_config):
        raise ValueError(f"{args.megatron_dataset_config=} does not exist")
    if args.batch_size is None:
        raise ValueError("batch_size must be specified")
    if isinstance(args.tags, str):
        args.tags = args.tags.split(",")

    if args.frozen_dtype not in (None, "bf16", "fp8", "fp8_full") and args.quantize is None:  # fp8 is a compute path of the fused executor
        args.quantize = args.frozen_dtype

    if args.relora and not args.use_peft:
        logger.warning("--relora assumes --use_peft. Setting --use_peft=True")
        args.use_peft = True
    if not args.use_peft:
        args.relora = None
        args.lora_r = None
        args.force_keep_original = False

    if args.total_batch_size is None:
        args.gradient_accumulation = args.gradient_accumulation or 1
        args.total_batch_size = args.batch_size * args.gradient_accumulation
    assert args.total_batch_size % args.batch_size == 0, "total_batch_size must be divisible by batch_size"

    if args.max_train_tokens is not None:
        # upstream divides *tokens* by *sequences* here (quirk kept under --parity_quirks)
        denom = args.total_batch_size if args.parity_quirks else args.total_batch_size * args.max_length
        args.num_training_steps = args.max_train_tokens // denom
        logger.info(f"Training for {args.num_training_steps} update steps")

    if args.warmed_up_model is not None:
        assert os.path.exists(args.warmed_up_model), f"{args.warmed_up_model=} does not exist"
    if args.dtype in ("fp16", "float16"):
        raise NotImplementedError("fp16 is not supported; use bfloat16 or float32")

    if (int(bool(args.reset_optimizer_on_relora)) + int(bool(args.optimizer_random_pruning))
            + int(bool(args.optimizer_magnitude_pruning))) > 1:
        raise ValueError("reset_optimizer_on_relora, optimizer_random_pruning and optimizer_magnitude_pruning are mutually exclusive")
    assert 0 <= args.optimizer_random_pruning < 1, "--optimizer_random_pruning must be between 0 and 1"
    assert 0 <= args.optimizer_magnitude_pruning < 1, "--optimizer_magnitude_pruning must be between 0 and 1"

    if args.relora is not None and args.cycle_length is None:
        logger.warning(f"cycle_length is not set for a ReLoRA run; defaulting to relora={args.relora}")
        args.cycle_length = args.relora

    if args.distributed_type == "fsdp" and args.weight_decay > 0:
        raise ValueError("FSDP does not support weight decay yet.")
    if args.distributed_type == "fsdp" and "zero" in args.optimizer.lower():
        raise ValueError("FSDP does zero-optimization by default, do not specify optimizer as zero optimizer.")

    if isinstance(args.skip_batches, str):
        args.skip_batches = set(map(int, args.skip_batches.split(",")))
        logger.info(f"Skipping batches {args.skip_batches}")
    args.skip_batches = set(args.skip_batches) if args.skip_batches else set()
    return args


def parse_args(argv: Optional[List[str]] = None) -> argparse.Namespace:
    parser = build_parser()
    args = parser.parse_args(argv)
    return check_args(args, argv)
