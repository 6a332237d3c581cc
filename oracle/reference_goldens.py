"""Record upstream outputs for the tests that compare this repo with the original ReLoRA code.

    python oracle/reference_goldens.py /path/to/upstream/relora

Each case builds this repo's seeded inputs exactly as its test does, copies the weights into the upstream model, and stores what
the upstream code computes on them:

* tests/golden/reference_models.json
    llama_9m            state-dict key set and shapes, a seeded logits sample, the loss, per-parameter gradient samples and norms
                        (tests/test_models.py::test_llama_matches_reference_logits_and_grads)
    padding_row         input-embedding gradient norms of a 12-layer llama_35m for a sequence starting with an ordinary token and
                        with the padding row (tests/test_models.py::test_sequence_starting_with_the_padding_row_...)
    relora_interchange  the upstream ReLoRaModel's state-dict layout, logits sample, loss and merged q / down projection samples
                        (tests/test_relora_core.py::test_reference_relora_state_dict_interchange)
* tests/golden/reference_schedulers.json
    the upstream LR lambdas at steps 0..199 (tests/test_schedulers.py::test_matches_reference_everywhere)
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import test_models as tm  # noqa: E402
import test_relora_core as trc  # noqa: E402
import test_schedulers as ts  # noqa: E402
from loss_curve_parity import import_upstream  # noqa: E402


def g9(x):
    """float32 data at float32 precision (9 significant digits): keeps the stored file small."""
    if isinstance(x, dict):
        return {k: g9(v) for k, v in x.items()}
    if isinstance(x, list):
        return [g9(v) for v in x]
    return float(f"{x:.9g}") if isinstance(x, float) else x


def shapes(sd):
    return {k: list(v.shape) for k, v in sd.items()}


def main(ref_root: str) -> None:
    from transformers import AutoConfig

    up = import_upstream(ref_root)
    cfg_dir = os.path.join(ref_root, "configs")
    out = {}

    # llama_9m logits / gradients
    ours, ids = tm.llama9m_case()
    ref = up.llama.LlamaForCausalLM(AutoConfig.from_pretrained(os.path.join(cfg_dir, "llama_9m.json")))
    ref.load_state_dict(ours.state_dict(), strict=True)
    a = ref(input_ids=ids, labels=ids)
    a.loss.backward()
    out["llama_9m"] = {
        "state_dict_shapes": shapes(ref.state_dict()),
        "logits_sample": tm.sample(a.logits, 512).tolist(), "loss": float(a.loss),
        "grad_samples": {n: tm.sample(p.grad, 16).tolist() for n, p in ref.named_parameters()},
        "grad_norms": {n: float(p.grad.double().norm()) for n, p in ref.named_parameters()},
    }

    # padding row overflow
    model, ids = tm.padding_row_case()
    hf_cfg = AutoConfig.from_pretrained(os.path.join(cfg_dir, "llama_35m.json"))
    hf_cfg.num_hidden_layers = 12
    ref = up.llama.LlamaForCausalLM(hf_cfg)
    ref.load_state_dict(model.state_dict(), strict=True)
    norms = tm.padding_row_grad_norms(ref, ids, ref.model.embed_tokens)
    out["padding_row"] = {"reference_grad_norms": {str(k): v for k, v in norms.items()}}

    # ReLoRA state-dict interchange + merge
    ours, ids = trc.relora_interchange_case()
    ref_w = up.relora.ReLoRaModel(up.llama.LlamaForCausalLM(AutoConfig.from_pretrained(os.path.join(cfg_dir, "llama_9m.json"))), r=8,
                                  lora_alpha=32, target_modules=trc.TARGETS, lora_dropout=0.1, keep_original_weights=True)
    ref_w.wrapped_model.load_state_dict(ours.wrapped_model.state_dict(), strict=True)
    ref_w.eval()
    with torch.no_grad():
        a = ref_w(input_ids=ids, labels=ids)
    idx = torch.randint(0, a.logits.numel(), (1024,), generator=torch.Generator().manual_seed(0))
    entry = {"state_dict_shapes": shapes(ref_w.wrapped_model.state_dict()),
             "logits_sample": a.logits.reshape(-1)[idx].double().tolist(), "loss": float(a.loss)}
    ref_w.merge_and_reinit()
    entry["merged_samples"] = trc.merged_samples(ref_w)
    out["relora_interchange"] = entry
    with open(os.path.join(ROOT, "tests", "golden", "reference_models.json"), "w") as f:
        json.dump(g9(out), f)
        f.write("\n")

    sched = {}
    for name, _, fn, kw in ts.REFERENCE_CASES:
        lam = getattr(up.training_utils, fn)
        sched[name] = [float(lam(s, **kw)) for s in range(200)]
    with open(os.path.join(ROOT, "tests", "golden", "reference_schedulers.json"), "w") as f:
        json.dump(sched, f)
        f.write("\n")
    print("padding-row norms", norms)


if __name__ == "__main__":
    main(sys.argv[1])
