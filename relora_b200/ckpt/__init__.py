"""Checkpointing in the reference's on-disk layout (SURVEY §5.4).

    <save_dir>/training_config.yaml
    <save_dir>/model_<update_step>/config.json, pytorch_model.bin [, relora_config.json]
                                   optimizer.pt          {optimizer, scheduler, update_step, global_step, config, dtype}
                                   training_state.json   {global_step, update_step, tokens_seen, tokens_seen_before,
                                                          n_lora_restarts, n_optimizer_resets, update_time, wandb_id}

Parity target: ``torchrun_main.py:192-273`` (save), ``:505-527`` (warm start), ``:555-583, 693-716``
(resume), ``training_utils.py:248-264`` (latest checkpoint), ``:406-418`` (retention).
"""
from __future__ import annotations

import json
import os
import shutil
import time
from typing import Any, Dict, Optional, Tuple

import torch
import yaml

from ..obs import logger

__all__ = [
    "save_checkpoint",
    "get_last_training_state",
    "delete_old_checkpoints",
    "load_model_weights",
    "load_training_state",
    "load_optimizer_checkpoint",
    "dump_training_config",
    "diff_training_config",
]


def _unwrap(model):
    return model.module if hasattr(model, "module") and isinstance(model.module, torch.nn.Module) else model


def save_checkpoint(
    model,
    *,
    optimizer,
    scheduler,
    training_state: Dict[str, Any],
    run_config: Dict[str, Any],
    save_dir: str,
    dtype: str,
    rank: int = 0,
    barrier=None,
    run_id: Optional[str] = None,
) -> float:
    """Write one ``model_<step>`` directory.  Rank 0 writes; ``barrier`` (if given) is called at the
    same two points as upstream.  Optimizers exposing ``consolidate_state_dict`` (ZeRO-style
    sharding) are consolidated on every rank before rank 0 serialises them."""
    t0 = time.time()
    if rank == 0:
        os.makedirs(save_dir, exist_ok=True)
        _unwrap(model).save_pretrained(save_dir)
    if barrier is not None:
        barrier()
    if hasattr(optimizer, "consolidate_state_dict"):
        optimizer.consolidate_state_dict()
    if rank == 0:
        payload = {
            "optimizer": optimizer.state_dict(),
            "scheduler": scheduler.state_dict(),
            "update_step": training_state["update_step"],
            "global_step": training_state["global_step"],
            "config": run_config,
            "dtype": dtype,
        }
        torch.save(payload, os.path.join(save_dir, "optimizer.pt"))
        state = dict(training_state)
        state["wandb_id"] = run_id
        with open(os.path.join(save_dir, "training_state.json"), "w") as f:
            json.dump(state, f, indent=4)
    dt = time.time() - t0
    logger.info(f"Saving took {dt:.2f} seconds")
    if barrier is not None:
        barrier()
    return dt


def _step_of(name: str) -> int:
    return int(name.split("_")[-1])


def get_last_training_state(save_dir: str) -> Tuple[Optional[dict], Optional[str]]:
    """Pick the ``model_<N>`` directory with the largest N and read its ``training_state.json``."""
    dirs = [d for d in os.listdir(save_dir) if d.startswith("model_")]
    if not dirs:
        logger.warning(f"Save directory {save_dir} exists, but does not contain any models.")
        logger.warning("Starting training from scratch.")
        return None, None
    last = os.path.join(save_dir, max(dirs, key=_step_of))
    logger.info(f"Restarting training from {last}")
    with open(os.path.join(last, "training_state.json")) as f:
        return json.load(f), last


def delete_old_checkpoints(save_dir: str, keep: Optional[int]) -> None:
    if keep is None:
        return
    dirs = sorted((d for d in os.listdir(save_dir) if d.startswith("model_")), key=_step_of)
    if len(dirs) <= keep:
        return
    for d in dirs[:-keep] if keep > 0 else dirs:
        path = os.path.join(save_dir, d)
        logger.info(f"Deleting checkpoint {path}")
        shutil.rmtree(path, ignore_errors=True)


def load_model_weights(module: torch.nn.Module, directory: str, strict: bool = True) -> None:
    """Load ``pytorch_model.bin`` (hard-coded name upstream), ``model.safetensors`` or a sharded checkpoint's ``*.index.json``.
    Hugging Face Llama checkpoints carry no ``rotary_emb.inv_freq`` buffers: those keep the module's values."""
    from ..models.llama import load_state_dict_files

    state = load_state_dict_files(directory)
    if hasattr(module, "load_hf_state_dict"):
        module.load_hf_state_dict(state, strict=strict)
    else:
        own = module.state_dict()
        state.update({k: v for k, v in own.items() if k.endswith("rotary_emb.inv_freq") and k not in state})
        module.load_state_dict(state, strict=strict)


def load_training_state(directory: str) -> Optional[dict]:
    path = os.path.join(directory, "training_state.json")
    if not os.path.exists(path):
        return None
    with open(path) as f:
        return json.load(f)


def load_optimizer_checkpoint(directory: str) -> dict:
    return torch.load(os.path.join(directory, "optimizer.pt"), map_location="cpu", weights_only=False)


def _yaml_safe(v):
    if isinstance(v, set):
        return sorted(v)
    if isinstance(v, tuple):
        return list(v)
    return v


def dump_training_config(args, save_dir: str) -> None:
    os.makedirs(save_dir, exist_ok=True)
    with open(os.path.join(save_dir, "training_config.yaml"), "w") as f:
        yaml.safe_dump({k: _yaml_safe(v) for k, v in vars(args).items()}, f)


def diff_training_config(args, save_dir: str) -> None:
    """Warn about every argument that changed since the run in ``save_dir`` was started."""
    path = os.path.join(save_dir, "training_config.yaml")
    if not os.path.exists(path):
        logger.warning(f"Training config not found in the existing save directory {save_dir}.")
        return
    with open(path) as f:
        old = yaml.safe_load(f) or {}
    new = {k: _yaml_safe(v) for k, v in vars(args).items()}
    if old != new:
        logger.warning("Arguments have changed since the last run.")
        logger.warning("Training config will be overwritten with new args")
        for k, v in new.items():
            if old.get(k) != v:
                logger.warning(f"{k:30} {old.get(k)} -> {v}")
