"""Record the upstream ReLoRA trainer's loss curve for tests/test_loss_curve_parity.py.

    python oracle/loss_curve_parity.py /path/to/upstream/relora [tests/golden/loss_curve_parity.json]

Builds this repo's llama_9m TrainingEngine exactly as the test does (seeded weights, live LoRA branch), copies those weights
into the upstream model / ReLoRaModel, drives it with the upstream scheduler / optimizer-reset code through the loop of
upstream torchrun_main.py:768-826 on the test's seeded batches, and stores the per-step losses together with a fingerprint of
the starting weights.  The test then compares this repo's losses with the stored curve without needing the upstream tree.
"""
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_loss_curve_parity import RELORA_EVERY, STEPS, batches, build_engine, weight_fingerprint  # noqa: E402

TARGETS = ["attn", "attention", "mlp"]


def import_upstream(ref_root: str):
    """The upstream modeling / relora / training_utils modules, with a stub ``bitsandbytes`` (imported at module level upstream;
    the fp32 paths never call it)."""
    bnb = types.ModuleType("bitsandbytes")
    bnb.nn, bnb.functional = types.ModuleType("bitsandbytes.nn"), types.ModuleType("bitsandbytes.functional")
    sys.modules.update({"bitsandbytes": bnb, "bitsandbytes.nn": bnb.nn, "bitsandbytes.functional": bnb.functional})
    if ref_root not in sys.path:
        sys.path.append(ref_root)
    import importlib

    return types.SimpleNamespace(llama=importlib.import_module("peft_pretraining.modeling_llama"),
                                 relora=importlib.import_module("peft_pretraining.relora"),
                                 training_utils=importlib.import_module("peft_pretraining.training_utils"))


def main(ref_root: str, out: str) -> None:
    from transformers import AutoConfig

    up = import_upstream(ref_root)
    ref_llama, ref_relora, tu = up.llama, up.relora, up.training_utils

    eng = build_engine()
    cfg = AutoConfig.from_pretrained(os.path.join(ROOT, "configs", "llama_9m.json"))
    ref_w = ref_relora.ReLoRaModel(ref_llama.LlamaForCausalLM(cfg), r=8, lora_alpha=32, target_modules=TARGETS, lora_dropout=0.0,
                                   keep_original_weights=True)
    ref_w.wrapped_model.load_state_dict(eng.model.wrapped_model.state_dict(), strict=True)
    trainable = [p for p in ref_w.parameters() if p.requires_grad]
    lora_params = [p for n, p in ref_w.named_parameters() if p.requires_grad and "lora_" in n]
    opt = torch.optim.AdamW(trainable, lr=1e-3, betas=(0.9, 0.999), weight_decay=0.0)
    sch = tu.get_scheculer(opt, scheduler_type="cosine_restarts", num_training_steps=9, warmup_steps=1, min_lr_ratio=0.1,
                           cycle_length=RELORA_EVERY, restart_warmup_steps=1)
    losses = []
    ref_w.train()
    for step, batch in enumerate(batches(cfg.vocab_size), start=1):
        tot = 0.0
        for i in range(batch.shape[0]):
            loss = ref_w(input_ids=batch[i], labels=batch[i].clone()).loss
            (loss / batch.shape[0]).backward()
            tot += float(loss.detach())
        torch.nn.utils.clip_grad_norm_(trainable, 1.0, error_if_nonfinite=True)
        opt.step()
        sch.step()
        opt.zero_grad()
        losses.append(tot / batch.shape[0])
        # upstream resets at update_step % relora == 1 (torchrun_main.py:877-912): merge, then prune the LoRA moments
        if step % RELORA_EVERY == 1 and step > 1:
            ref_w.merge_and_reinit()
            tu.optimizer_reset(opt, reset_params=lora_params, optimizer_state_keys=["exp_avg", "exp_avg_sq"],
                               reset_optimizer_on_relora=False, optimizer_random_pruning=0.0, optimizer_magnitude_pruning=0.9)
    assert len(losses) == STEPS
    with open(out, "w") as f:
        json.dump({"weight_fingerprint": weight_fingerprint(eng), "reference_losses": losses}, f, indent=1)
        f.write("\n")
    print(out, losses)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "tests", "golden", "loss_curve_parity.json"))
