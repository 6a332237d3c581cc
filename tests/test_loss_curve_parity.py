"""Loss-curve parity with the unmodified reference on synthetic tokens (CPU, fp32, llama_9m): same initial weights, same
batches, the reference's own model / ReLoRaModel / scheduler / optimizer-reset code driven by the loop of
``torchrun_main.py:768-826`` versus this repo's TrainingEngine (SURVEY.md §4: "reference-vs-new loss-curve parity").

The reference side is stored in tests/golden/loss_curve_parity.json (recorded by oracle/loss_curve_parity.py from this
engine's starting weights), so the comparison runs without the reference tree."""
import json
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "loss_curve_parity.json")
STEPS, RELORA_EVERY, GA, B, T = 7, 3, 2, 2, 32


def build_engine():
    from relora_b200.engine.api import TrainingEngine

    torch.manual_seed(0)
    eng = TrainingEngine.build(
        model_config=os.path.join(ROOT, "configs", "llama_9m.json"), batch_size=B, gradient_accumulation=GA, total_batch_size=B * GA,
        max_length=T, use_peft=True, lora_r=8, lora_alpha=32, lora_dropout=0.0, relora=RELORA_EVERY, cycle_length=RELORA_EVERY,
        scheduler="cosine_restarts", warmup_steps=1, restart_warmup_steps=1, lr=1e-3, num_training_steps=9, dtype="float32", device="cpu",
        reset_optimizer_on_relora=False, optimizer_magnitude_pruning=0.9, clip_grad_norm=1.0, min_lr_ratio=0.1)
    # make the LoRA branch live from the start (upstream starts with A = B = 0)
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for n, p in sorted(eng.model.wrapped_model.named_parameters()):
            if "lora_" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
    return eng


def batches(vocab_size):
    g = torch.Generator().manual_seed(1)
    return [torch.randint(0, vocab_size, (GA, B, T), generator=g) for _ in range(STEPS)]


def weight_fingerprint(eng):
    """Per-tensor sums of the starting weights: tells a changed initialisation apart from a changed training step."""
    return {n: float(t.double().sum()) for n, t in sorted(eng.model.wrapped_model.state_dict().items())}


def test_training_losses_match_the_reference_through_a_relora_reset():
    golden = json.load(open(GOLDEN))
    eng = build_engine()
    fp = weight_fingerprint(eng)
    assert fp.keys() == golden["weight_fingerprint"].keys()
    for n, v in fp.items():
        assert abs(v - golden["weight_fingerprint"][n]) <= 1e-6 * max(1.0, abs(v)), f"starting weights differ from the recorded run: {n}"
    ref_losses = golden["reference_losses"]
    our_losses = [float(eng.train_step(batch)) for batch in batches(eng.model.config.vocab_size)]
    # identical until (and including) the first update after the merge: the merged weights agree and B = 0 on both sides;
    # afterwards the re-initialised A differs by construction (upstream draws it from the torch generator, we hash)
    n_exact = RELORA_EVERY + 2
    for a, b in zip(ref_losses[:n_exact], our_losses[:n_exact]):
        assert abs(a - b) < 2e-4, (ref_losses, our_losses)
    assert eng.n_lora_restarts >= 1
    # later steps: same trajectory up to the different (but equally distributed) re-initialisation
    for a, b in zip(ref_losses[n_exact:], our_losses[n_exact:]):
        assert abs(a - b) < 0.05, (ref_losses, our_losses)
