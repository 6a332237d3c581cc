"""Training orchestration: init, hot loop, evaluation, checkpoint/resume, ReLoRA reset schedule.

Parity target: reference ``torchrun_main.py:338-1018`` (``main``) and ``:143-189``
(``evaluate_model``).  Control flow, counters, reset conditions and the checkpoint layout follow the
reference step for step; what differs is *how* a step executes:

* gradients are reduced once per update, not once per micro-batch (see ``parallel.grad_sync``);
* the step itself runs through a stepper (``engine.stepper`` / ``engine.fused_llama``);
* throughput is device-timed with CUDA events and reported as the max over ranks
  (upstream: host ``time.time()``, ``:750, 826, 943``);
* the backend is NCCL on GPUs and gloo on CPU, so the same loop is testable without a GPU.
"""
from __future__ import annotations

import gc
import math
import os
import random
import time
from dataclasses import asdict, dataclass
from typing import Optional

import numpy as np
import torch
import torch.distributed as dist

from .. import ckpt as ckpt_lib
from ..data import (SkipDataLoader, SyntheticTokens, check_dataset_size, collate_input_ids, load_pretokenized,
                    shard_for_rank)
from ..models import LlamaForCausalLM, config_to_dict, load_config
from ..models.pythia import GPTNeoXForCausalLM
from ..obs import JsonlSink, PhaseTimer, logger, make_sink, maybe_make_profiler, silence_non_zero_rank
from ..parallel.dist import barrier, broadcast_object, init_distributed, shutdown
from ..relora import ReLoRaLinear, ReLoRaModel
from .stepper import make_scheduler, make_stepper, reset_optimizer, wrap_relora

__all__ = ["run", "evaluate_model", "TrainState"]


@dataclass
class TrainState:
    global_step: int = 0
    update_step: int = 0
    tokens_seen: int = 0
    tokens_seen_before: int = 0
    n_lora_restarts: int = 0
    n_optimizer_resets: int = 0


class _DeviceTimer:
    """CUDA-event timer on GPU (device time), ``perf_counter`` on CPU."""

    def __init__(self, device: torch.device):
        self.cuda = device.type == "cuda"
        self._t0 = None
        if self.cuda:
            self._e0 = torch.cuda.Event(enable_timing=True)
            self._e1 = torch.cuda.Event(enable_timing=True)

    def start(self):
        if self.cuda:
            self._e0.record()
        else:
            self._t0 = time.perf_counter()

    def stop_s(self) -> float:
        if self.cuda:
            self._e1.record()
            self._e1.synchronize()
            return self._e0.elapsed_time(self._e1) / 1e3
        return time.perf_counter() - self._t0


def pretrained_model(path: str, revision: Optional[str] = None):
    """The model of a local checkpoint directory, by the ``model_type`` of its ``config.json``: ``llama`` (Llama-family
    checkpoints, grouped-query attention included) or ``gpt_neox`` (Pythia)."""
    cfg_file = os.path.join(path, "config.json")
    if os.path.isdir(path) and os.path.exists(cfg_file):
        import json

        with open(cfg_file) as f:
            model_type = json.load(f).get("model_type")
        if model_type == "llama":
            return LlamaForCausalLM.from_pretrained(path)
        if model_type != "gpt_neox":
            raise NotImplementedError(f"model_type {model_type!r} in {cfg_file}: only llama and gpt_neox checkpoints are supported")
    return GPTNeoXForCausalLM.from_pretrained(path, revision=revision)


def _max_over_ranks(x: float, device) -> float:
    if dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.tensor([x], dtype=torch.float64, device=device if device.type == "cuda" else "cpu")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())
    return x


@torch.no_grad()
def evaluate_model(stepper, eval_loader, device, target_eval_tokens: int = 10_000_000):
    """Mean of per-batch losses over ~``target_eval_tokens`` tokens (-1 = whole set), all-reduced.

    Reference ``torchrun_main.py:143-189``.  The model is always returned to train mode (upstream's
    ``was_training = model.train`` is a bound method and therefore truthy).
    """
    t0 = time.time()
    model = stepper.model
    model.eval()
    acc = torch.zeros(3, dtype=torch.float64, device=device)  # Σ loss, batches, tokens
    n_eval_iters = None
    for i, batch in enumerate(eval_loader):
        ids = batch["input_ids"]
        if i == 0:
            tok = torch.tensor([float(ids.numel())], dtype=torch.float64, device=device)
            if dist.is_initialized() and dist.get_world_size() > 1:
                dist.all_reduce(tok)
            n_eval_iters = int(target_eval_tokens / tok.item())
        if target_eval_tokens != -1 and i > n_eval_iters:
            break
        ids = ids.to(device, non_blocking=True)
        loss = stepper.eval_loss(ids)
        acc[0] += loss.double()
        acc[1] += 1
        acc[2] += ids.numel()
    if torch.isnan(acc[0]):
        raise RuntimeError(f"Rank {dist.get_rank() if dist.is_initialized() else 0} got nan loss. This is probably a bug.")
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(acc)
    eval_loss = (acc[0] / acc[1].clamp(min=1)).float()
    tokens = acc[2].item()
    logger.info(f"Evaluated on {tokens} tokens, eval loss: {eval_loss:.4f}")
    logger.info(f"Evaluation took {time.time() - t0:.2f} seconds")
    model.train()
    return eval_loss, tokens


def _build_data(args, info, state_update_step: int):
    """Return ``(train_loader, eval_loader, test_loader, prep_args, vocab_size_or_None)``."""
    if args.synthetic_data is not None:
        n = int(args.synthetic_data)
        cfg = load_config(args.model_config or args.model_name_or_path)
        train = SyntheticTokens(n, args.max_length, cfg.vocab_size, seed=args.seed + 1)
        val = SyntheticTokens(max(args.batch_size * info.world_size * 2, 64), args.max_length, cfg.vocab_size, seed=args.seed + 2)
        check_dataset_size(len(train), args.max_length, args.total_batch_size, args.num_training_steps, args.parity_quirks)
        train, val = train.shard(info.rank, info.world_size), val.shard(info.rank, info.world_size)
        prep = {"tokenizer": "synthetic", "sequence_length": args.max_length}
        vocab = None
    elif args.dataset_path is not None:
        logger.info("Loading Huggingface dataset from directory")
        train, val, prep = load_pretokenized(args.dataset_path, seed=args.seed)
        logger.info("Checking datasets size")
        check_dataset_size(len(train), args.max_length, args.total_batch_size, args.num_training_steps, args.parity_quirks)
        assert prep["sequence_length"] == args.max_length
        vocab = prep.get("vocab_size")
        if vocab is None:
            try:
                from transformers import AutoTokenizer

                vocab = AutoTokenizer.from_pretrained(prep["tokenizer"], model_max_length=args.max_length).vocab_size
            except Exception as e:
                logger.warning(f"Could not load tokenizer {prep['tokenizer']!r} ({type(e).__name__}); skipping the vocab-size check")
        logger.info(f"Full training set size: {len(train)}")
        train, val = shard_for_rank(train, info.rank, info.world_size), shard_for_rank(val, info.rank, info.world_size)
        logger.info(f"Train set size after shard: {len(train)}")
    else:
        from ..data.neox import load_megatron_dataset

        start_iteration = 0
        if args.model_revision is not None and str(args.model_revision).startswith("step"):
            start_iteration = int(args.model_revision[4:])
            logger.info(f"Starting from iteration {start_iteration} based on model revision {args.model_revision}")
        tl, el, tsl, tok_name, vocab = load_megatron_dataset(args, world_size=info.world_size, rank=info.rank,
                                                            start_iteration=start_iteration)
        return tl, el, tsl, {"tokenizer": tok_name}, vocab

    skip = state_update_step * args.gradient_accumulation
    logger.info(f"Skipping the first {skip} batches")
    pin = info.device.type == "cuda"
    workers = args.workers if args.synthetic_data is None else 0
    train_loader = SkipDataLoader(train, batch_size=args.batch_size, collate_fn=collate_input_ids, skip_batches=skip,
                                  num_workers=workers, pin_memory=pin)
    eval_loader = torch.utils.data.DataLoader(val, batch_size=args.batch_size, collate_fn=collate_input_ids,
                                              num_workers=workers, pin_memory=pin)
    return train_loader, eval_loader, None, prep, vocab


def _dropout_seed_value(device):
    """Current value of the device-resident LoRA-dropout counter (None on CPU, where torch's generator is used)."""
    if device.type != "cuda":
        return None
    from ..ops import fused as _f

    return _f.seed_value(device)


def run(args) -> dict:
    """Train according to ``args`` (a namespace from :func:`relora_b200.config.parse_args`)."""
    torch.manual_seed(args.seed)
    np.random.seed(args.seed)
    random.seed(args.seed)

    info = init_distributed(args.device, args.backend)
    device, rank, world = info.device, info.rank, info.world_size
    logger.info(f"Global rank {rank}, local rank {info.local_rank}, device: {device}, backend {info.backend}")

    if args.distributed_type == "fsdp":
        raise RuntimeError("FSDP is not supported anymore. There were a lot of isses with ReLoRA and FSDP "
                           "and no speed or memory improvements.")

    if args.total_batch_size is not None and args.gradient_accumulation is None:
        assert args.total_batch_size % world == 0, "total_batch_size must be divisible by world_size"
        args.gradient_accumulation = args.total_batch_size // (args.batch_size * world)
        assert args.gradient_accumulation > 0, "gradient_accumulation must be greater than 0"
    assert args.gradient_accumulation * args.batch_size * world == args.total_batch_size, \
        "gradient_accumulation * batch_size * world_size must be equal to total_batch_size"
    if args.max_train_tokens is not None:
        denom = args.total_batch_size if args.parity_quirks else args.total_batch_size * args.max_length
        args.num_training_steps = args.max_train_tokens // denom
        logger.info(f"Setting num_training_steps to {args.num_training_steps} based on max_train_tokens")

    silence_non_zero_rank(rank)

    # ---------------------------------------------------------------- autoresume
    run_id = None
    if args.save_dir is not None and os.path.exists(args.save_dir):
        if not args.autoresume:
            raise ValueError(f"Save directory {args.save_dir} already exists and --autoresume is off. Interrupting...")
        ckpt_lib.diff_training_config(args, args.save_dir)
        training_state, resume_from = ckpt_lib.get_last_training_state(args.save_dir)
        if args.resume_from is None:
            args.resume_from = resume_from
        if training_state is not None:
            run_id = training_state.get("wandb_id")
        logger.info(f"Resuming training from {resume_from} with wandb id {run_id}")
    barrier()

    sink = None
    if rank == 0:
        sink = make_sink(tags=args.tags, run_id=run_id, notes=args.comment)
        args.run_name = sink.name
        if args.save_dir is None:
            args.save_dir = f"checkpoints/{sink.name}"
        os.makedirs(args.save_dir, exist_ok=True)
        if isinstance(sink, JsonlSink):
            sink.attach(args.save_dir)
        ckpt_lib.dump_training_config(args, args.save_dir)
    barrier()
    args.run_name = broadcast_object(getattr(args, "run_name", None))
    if args.save_dir is None:
        args.save_dir = f"checkpoints/{args.run_name}"

    logger.info("*" * 40)
    logger.info("Starting training with the arguments")
    for k, v in vars(args).items():
        logger.info(f"{k:30} {v}")
    logger.info("*" * 40)

    st = TrainState()

    # ---------------------------------------------------------------- model
    if args.model_config is not None:
        model_config = load_config(args.model_config)
        if getattr(model_config, "model_type", "llama") != "llama":
            raise NotImplementedError(f"Unknown model config type {type(model_config)}, only LLaMA is supported")
        model = LlamaForCausalLM(model_config)
    else:
        logger.info(f"Using pretrained model {args.model_name_or_path} revision {args.model_revision}")
        model = pretrained_model(args.model_name_or_path, args.model_revision)
        model_config = model.config

    if args.warmed_up_model is not None:
        logger.info("*" * 40)
        logger.info(f"Loading a warmed-up model from {args.warmed_up_model}")
        ckpt_lib.load_model_weights(model, args.warmed_up_model, strict=True)
        old = ckpt_lib.load_training_state(args.warmed_up_model)
        if old is not None:
            st.global_step, st.update_step = old["global_step"], old["update_step"]
            st.tokens_seen, st.tokens_seen_before = old["tokens_seen"], old["tokens_seen_before"]
            logger.info(f"global_step {st.global_step}, update_step {st.update_step}, tokens_seen {st.tokens_seen}")
            logger.info(f"Will train for {args.num_training_steps - st.update_step} update steps")
        else:
            logger.warning(f"Did not find training state in {args.warmed_up_model}, global step will start from zero")
        logger.info("*" * 40)

    params_before = sum(p.numel() for p in model.parameters())
    if args.use_peft:
        need_linear_weight = args.relora is not None or args.force_keep_original or args.warmed_up_model is not None
        logger.info(f"Wrapping model with LoRA ({need_linear_weight=})")
        model = wrap_relora(model, args, lora_only=not need_linear_weight)

    _update_step_ckpt = None
    _resume_dropout_seed = None
    if args.resume_from:
        logger.info(f"Loading model from {args.resume_from}")
        target = model.wrapped_model if isinstance(model, ReLoRaModel) else model
        ckpt_lib.load_model_weights(target, args.resume_from, strict=True)
        old = ckpt_lib.load_training_state(args.resume_from)
        st.global_step = old["global_step"]
        _update_step_ckpt = old["update_step"]  # not applied here: the scheduler must start from the warm-start step
        st.tokens_seen, st.tokens_seen_before = old["tokens_seen"], old["tokens_seen_before"]
        st.n_lora_restarts = old.get("n_lora_restarts", 0)
        st.n_optimizer_resets = old.get("n_optimizer_resets", 0)
        _resume_dropout_seed = old.get("dropout_seed")
        if isinstance(model, ReLoRaModel):
            model.n_restarts = st.n_lora_restarts
        logger.info(f"Will train for {args.num_training_steps - _update_step_ckpt} update steps")

    params_after = sum(p.numel() for p in model.parameters())
    logger.info(f"\n{model}\n")
    logger.info(f"Total params  before LoRA: {params_before / 1e6:.2f}M")
    logger.info(f"Total params  after  LoRA: {params_after / 1e6:.2f}M")
    logger.info(f"Trainable params: {sum(p.numel() for p in model.parameters() if p.requires_grad) / 1e6:.2f}M")
    logger.info(f"In total, added {(params_after - params_before) / 1e6:.2f}M parameters to the model")
    logger.info(f"Saving model to {args.save_dir} every {args.save_every} update steps")

    if args.dtype in ("bf16", "bfloat16"):
        model = model.to(device=device, dtype=torch.bfloat16)
    else:
        model = model.to(device=device)

    n_total = sum(p.numel() for p in model.parameters())
    n_train = sum(p.numel() for p in model.parameters() if p.requires_grad)

    # ---------------------------------------------------------------- data (after the model: vocab check)
    train_loader, eval_loader, test_loader, prep_args, data_vocab = _build_data(args, info, 0)
    if data_vocab is not None and args.model_config is not None and model_config.vocab_size != data_vocab:
        logger.warning(f"Model config vocab size ({model_config.vocab_size}) does not match tokenizer vocab size ({data_vocab})")
        if not (model_config.vocab_size == 32000 and data_vocab == 32100) and model_config.vocab_size < data_vocab:
            raise ValueError(f"Model config vocab size ({model_config.vocab_size}) does not match tokenizer vocab size ({data_vocab})")

    # ---------------------------------------------------------------- executor / optimizer / scheduler
    # a resumed run continues the LoRA-dropout stream from the counter saved in training_state.json instead of replaying the masks
    # of step 0
    stepper = make_stepper(model, info, args, dropout_seed=_resume_dropout_seed)
    optimizer = stepper.optimizer
    lora_params = stepper.lora_params
    if args.use_peft and len(lora_params) == 0:
        raise ValueError("No LoRA parameters found")

    run_config = dict(vars(args))
    run_config["skip_batches"] = sorted(run_config.get("skip_batches") or [])
    run_config.update({
        "tokenizer": prep_args["tokenizer"],
        "max_lr": run_config.pop("lr"),
        "total_params_M": n_total / 1e6,
        "trainable_params_M": n_train / 1e6,
        "equivalent_params_M": params_before / 1e6,
        "percent_trainable_params": n_train / n_total,
        "name_trainable_params": stepper.trainable_names,
        "model": config_to_dict(model_config),
        "world_size": world,
        "device": str(device),
        "dataset_preprocessing_args": prep_args,
        "executor": type(stepper).__name__,
    })
    if rank == 0:
        sink.config_update(run_config)
        if args.wandb_watch:
            sink.watch(model, log_freq=500)

    scheduler_start_step = st.update_step
    sched_steps = args.num_training_steps - scheduler_start_step
    logger.info(f"Scheduler will run for {sched_steps} update steps")
    scheduler = make_scheduler(optimizer, args, sched_steps)

    if args.resume_from:
        # upstream replays `update_step` scheduler steps here with update_step still at the warm-start
        # value, then overwrites everything from optimizer.pt (torchrun_main.py:693-708)
        for _ in range(st.update_step):
            scheduler.step()
        if args.load_optimizer_state_on_resume:
            oc = ckpt_lib.load_optimizer_checkpoint(args.resume_from)
            optimizer.load_state_dict(oc["optimizer"])
            scheduler.load_state_dict(oc["scheduler"])
            st.update_step, st.global_step = oc["update_step"], oc["global_step"]
            logger.info(f"Optimizer and scheduler restored from {args.resume_from}")
        elif _update_step_ckpt is not None:
            pass  # keep upstream behaviour: counters stay at the warm-start values
        old_cfg_path = os.path.join(os.path.dirname(os.path.normpath(args.resume_from)), "training_config.yaml")
        for cand in (os.path.join(args.resume_from, "training_config.yaml"), old_cfg_path):
            if os.path.exists(cand):
                import yaml

                with open(cand) as f:
                    old_cfg = yaml.safe_load(f) or {}
                if old_cfg.get("batch_size") not in (None, args.batch_size):
                    raise RuntimeError("Cannot resume from a checkpoint with a different batch size.")
                break

    # rebuild the train loader with the resume offset now that update_step is final
    if st.update_step > 0 and args.megatron_dataset_config is None:
        train_loader, eval_loader, test_loader, _, _ = _build_data(args, info, st.update_step)
    elif args.megatron_dataset_config is not None and args.resume_from:
        train_loader.batch_sampler.start_iter = st.global_step

    # ---------------------------------------------------------------- loop
    timer = _DeviceTimer(device)
    phases = PhaseTimer()
    local_step = 0
    n_skipped = 0
    loss_acc = torch.zeros(3, dtype=torch.float32, device=device)  # Σ loss, batches, NaNs
    ga = args.gradient_accumulation
    prof = maybe_make_profiler(args.profile, args.run_name, rank)
    last_loss = None
    update_time = 0.0

    logger.info(f"Starting training at update step {st.update_step} with {args.num_training_steps - st.update_step} update steps")
    pbar = None
    if rank == 0:
        try:
            from tqdm import tqdm

            pbar = tqdm(total=args.num_training_steps - st.update_step, desc="Update steps", ncols=80,
                        disable=not os.isatty(2))
        except Exception:  # pragma: no cover
            pbar = None

    timer.start()
    exhausted = True
    for batch in train_loader:
        st.global_step += 1
        local_step += 1

        if st.update_step in args.skip_batches:
            if st.global_step % ga == 0:
                st.update_step += 1
            continue
        if local_step == 1:
            logger.info("Starting first step")
        if st.update_step >= args.num_training_steps:
            logger.info(f"Reached max number of update steps (f{args.num_training_steps}). Stopping training.")
            exhausted = False
            break

        ids = batch["input_ids"].to(device, non_blocking=True)
        st.tokens_seen += ids.numel() * world

        loss = stepper.micro_step(ids)
        loss_acc[0] += loss.float()
        loss_acc[1] += 1
        loss_acc[2] += torch.isnan(loss).float()

        if st.global_step % ga != 0:
            continue

        # ------------------------------------------------ update step
        if pbar is not None:
            pbar.update(1)
        if world > 1:
            dist.all_reduce(loss_acc, op=dist.ReduceOp.SUM)
        mean_loss = loss_acc[0] / loss_acc[1]
        has_nan = loss_acc[2] > 0
        uinfo = stepper.update(skip=has_nan, error_if_nonfinite=bool(args.clip_grad_norm > 0 and args.parity_quirks))
        skipped = bool(has_nan)  # one host sync per update (upstream has two: grad_norm.item() and this)
        if not skipped and not math.isfinite(float(uinfo.grad_norm)):
            # upstream dies here (clip_grad_norm_(error_if_nonfinite=True), reproduced under --parity_quirks); the kernels have
            # skipped the update on the device, so the run continues and the event is counted like a NaN loss
            logger.error(f"Non-finite gradient norm ({float(uinfo.grad_norm)}) at update {st.update_step}, skipping update")
            skipped = True
        if not skipped:
            scheduler.step()
        elif bool(has_nan):
            logger.error(f"Nan detected in loss_info, loss={float(mean_loss)}, skipping update")
        if skipped:
            if device.type == "cuda" and hasattr(optimizer, "rollback_skipped_step"):
                optimizer.rollback_skipped_step()  # the device-side skip left the moments untouched; undo the optimistic step count
            n_skipped += 1
            if n_skipped > 0.05 * args.num_training_steps:
                logger.error("More than 5% of batches skipped due to NaNs, stopping training.")
                exhausted = False
                break
        st.update_step += 1
        update_time = _max_over_ranks(timer.stop_s(), device)
        last_loss = float(mean_loss)
        grad_norm = float(uinfo.grad_norm)
        loss_acc.zero_()

        if local_step > ga and st.update_step % args.save_every == 0:
            directory = f"{args.save_dir}/model_{st.update_step}"
            logger.info(f"Saving model and optimizer to {directory}, update step {st.update_step}")
            with phases.phase("save"):
                ts = asdict(st)
                ts["update_time"] = update_time
                if device.type == "cuda":  # engine extension (readers of the reference layout ignore unknown keys)
                    ts["dropout_seed"] = _dropout_seed_value(device)
                ckpt_lib.save_checkpoint(model, optimizer=optimizer, scheduler=scheduler, training_state=ts,
                                         run_config=run_config, save_dir=directory, dtype=args.dtype, rank=rank,
                                         barrier=barrier, run_id=sink.id if sink else None)
                if args.keep_checkpoints is not None and rank == 0:
                    ckpt_lib.delete_old_checkpoints(args.save_dir, keep=args.keep_checkpoints)

        if st.update_step % args.eval_every == 0:
            logger.info(f"Performing evaluation at step {st.update_step}")
            with phases.phase("eval"):
                total_loss, evaluated_on = evaluate_model(stepper, eval_loader, device)
            if rank == 0:
                sink.log({"final_eval_loss": float(total_loss), "final_eval_tokens": evaluated_on}, step=st.global_step)
            logger.info(f"Eval loss at step {st.update_step}: {total_loss}")

        # ------------------------------------------------ ReLoRA merge + optimizer reset
        rel = st.update_step - scheduler_start_step
        can_reset_relora = args.relora is not None and (args.resume_from is not None or local_step // ga >= args.relora)
        if can_reset_relora and rel % args.relora == 1:
            t0 = time.time()
            logger.info(f"{args.resume_from=}, {local_step=}, {args.relora=}, thresh: {local_step // ga}")
            logger.info(f"Performing lora reset at update step {st.update_step}. Current lr is {optimizer.param_groups[0]['lr']}")
            st.n_lora_restarts += 1
            with phases.phase("merge"):
                stepper.merge_and_reinit()
            logger.info(f"LoRA reset took {time.time() - t0:.2f}s")

        can_reset_optimizer = args.relora is not None and (args.resume_from is not None or local_step // ga >= args.cycle_length)
        if can_reset_optimizer and rel % args.cycle_length == 1:
            logger.info(f"Performing optimizer reset at update step {st.update_step}. Current lr is {optimizer.param_groups[0]['lr']}")
            st.n_optimizer_resets += 1
            reset_optimizer(optimizer, lora_params, args, st.n_optimizer_resets)
            from ..utils import check_lr_and_alert, optimizer_state_size

            # after a reset the schedule must be at (nearly) zero lr; a large value means reset and schedule are out of phase
            check_lr_and_alert(optimizer, max_lr=0.05 * args.lr + 1e-12, sink=sink if rank == 0 else None, step=st.global_step)
            sz = optimizer_state_size(optimizer)
            logger.info(f"Optimizer state after reset: {sz['exp_avg_nonzero'] / 1e6:.2f}M / {sz['exp_avg_numel'] / 1e6:.2f}M non-zero first moments")
        if can_reset_optimizer and rel % args.cycle_length == 2:
            logger.info(f"First step after optimizer reset lr is {optimizer.param_groups[0]['lr']}")

        lr = optimizer.param_groups[0]["lr"]
        tokens_in_update = st.tokens_seen - st.tokens_seen_before
        st.tokens_seen_before = st.tokens_seen
        if rank == 0 and (st.update_step % max(1, args.log_every) == 0):
            sink.log({
                "loss": last_loss,
                "lr": lr,
                "grad_norm": grad_norm,
                "update_step": st.update_step,
                "tokens_seen": st.tokens_seen,
                "throughput_tokens": tokens_in_update / max(update_time, 1e-9),
                "throughput_examples": args.total_batch_size / max(update_time, 1e-9),
                "throughput_batches": ga * world / max(update_time, 1e-9),
                "n_lora_restarts": st.n_lora_restarts,
                "n_optimizer_resets": st.n_optimizer_resets,
            }, step=st.global_step)
            if args.train_scaling:
                scal = [float(m.scaling.data.item()) for m in model.modules() if isinstance(m, ReLoRaLinear)]
                sink.log({"lora_scaling": scal}, step=st.global_step)
        timer.start()
        if prof is not None:
            prof.step()
    else:
        pass
    if exhausted and st.update_step < args.num_training_steps:
        print(f"Warning: reached the end of the dataset. Training stopped, global_rank={rank}, update_step={st.update_step}")
        logger.warning("Reached the end of the dataset. Training stopped")

    if prof is not None:
        prof.stop()
    logger.info("Training finished")
    if pbar is not None:
        pbar.close()

    directory = f"{args.save_dir}/model_{st.update_step}"
    if not os.path.exists(directory):
        logger.info(f"Saving model and optimizer to {directory}, update step {st.update_step}")
        ts = asdict(st)  # incl. n_optimizer_resets (upstream drops it from the final checkpoint; the prune RNG is keyed by it)
        ts["update_time"] = update_time
        if device.type == "cuda":
            ts["dropout_seed"] = _dropout_seed_value(device)
        ckpt_lib.save_checkpoint(model, optimizer=optimizer, scheduler=scheduler, training_state=ts,
                                 run_config=run_config, save_dir=directory, dtype=args.dtype, rank=rank,
                                 barrier=barrier, run_id=sink.id if sink else None)
    else:
        barrier()

    logger.info("Running final evaluation")
    gc.collect()
    if device.type == "cuda":
        torch.cuda.empty_cache()
    final_loss, final_tokens = evaluate_model(stepper, eval_loader, device, target_eval_tokens=100_000_000)
    result = {"final_eval_loss": float(final_loss), "final_eval_tokens": final_tokens, "update_step": st.update_step,
              "global_step": st.global_step, "tokens_seen": st.tokens_seen, "last_train_loss": last_loss, "save_dir": args.save_dir,
              "n_lora_restarts": st.n_lora_restarts, "n_optimizer_resets": st.n_optimizer_resets,
              "executor": type(stepper).__name__}
    if rank == 0:
        sink.log({"final_eval_loss": float(final_loss), "final_eval_tokens": final_tokens}, step=st.global_step)
        logger.info(f"Final eval loss: {final_loss}")
    if test_loader is not None:
        logger.info("Running test evaluation (full test set!)")
        test_loss, test_tokens = evaluate_model(stepper, test_loader, device, target_eval_tokens=-1)
        result.update({"final_test_loss": float(test_loss), "final_test_tokens": test_tokens})
        if rank == 0:
            sink.log({"final_test_loss": float(test_loss), "final_test_tokens": test_tokens}, step=st.global_step)
            logger.info(f"Test loss: {test_loss}")
    if rank == 0:
        sink.finish()
    logger.info("Script finished successfully")
    print(f"Rank {rank} finished successfully")
    shutdown(info)
    return result
