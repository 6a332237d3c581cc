"""Model-config loading: HF ``LlamaConfig`` / ``GPTNeoXConfig`` JSON files and directories.

The reference reads ``configs/llama_*.json`` through ``AutoConfig.from_pretrained``
(``torchrun_main.py:478``).  Those files carry ``max_sequence_length`` rather than
``max_position_embeddings`` so the HF default of 2048 positions applies (SURVEY C14) — preserved.
"""
from __future__ import annotations

import copy
import json
import os
from typing import Any, Dict

__all__ = ["load_config", "save_config", "SimpleConfig", "config_to_dict", "rope_settings", "rope_scaling"]

_LLAMA_DEFAULTS = dict(
    model_type="llama",
    vocab_size=32000,
    hidden_size=4096,
    intermediate_size=11008,
    num_hidden_layers=32,
    num_attention_heads=32,
    hidden_act="silu",
    max_position_embeddings=2048,
    initializer_range=0.02,
    rms_norm_eps=1e-6,
    use_cache=True,
    pad_token_id=None,
    bos_token_id=1,
    eos_token_id=2,
    tie_word_embeddings=False,
    rope_theta=10000.0,
)

_NEOX_DEFAULTS = dict(
    model_type="gpt_neox",
    vocab_size=50432,
    hidden_size=6144,
    num_hidden_layers=44,
    num_attention_heads=64,
    intermediate_size=24576,
    hidden_act="gelu",
    rotary_pct=0.25,
    rotary_emb_base=10000,
    attention_dropout=0.0,
    hidden_dropout=0.0,
    classifier_dropout=0.1,
    max_position_embeddings=2048,
    initializer_range=0.02,
    layer_norm_eps=1e-5,
    use_cache=True,
    bos_token_id=0,
    eos_token_id=2,
    tie_word_embeddings=False,
    use_parallel_residual=True,
    rope_scaling=None,
    attention_bias=True,
)


class SimpleConfig:
    """Attribute bag with HF-like ``to_dict`` / ``save_pretrained`` (used when transformers is absent
    or for tests that should not depend on its version)."""

    def __init__(self, **kw):
        mt = kw.get("model_type", "llama")
        base = _NEOX_DEFAULTS if mt == "gpt_neox" else _LLAMA_DEFAULTS
        for k, v in base.items():
            setattr(self, k, v)
        for k, v in kw.items():
            setattr(self, k, v)
        if mt == "llama" and getattr(self, "num_key_value_heads", None) is None:
            self.num_key_value_heads = self.num_attention_heads  # multi-head attention unless the config says otherwise

    def to_dict(self) -> Dict[str, Any]:
        return copy.deepcopy(self.__dict__)

    def to_json_string(self) -> str:
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"

    def save_pretrained(self, directory: str):
        os.makedirs(directory, exist_ok=True)
        with open(os.path.join(directory, "config.json"), "w") as f:
            f.write(self.to_json_string())

    def __repr__(self):
        return f"SimpleConfig({self.to_dict()})"


def _resolve(path: str) -> str:
    if os.path.isdir(path):
        return os.path.join(path, "config.json")
    return path


def load_config(path: str, prefer_hf: bool = True):
    """Load a model config from a JSON file or a checkpoint directory."""
    file = _resolve(path)
    with open(file) as f:
        raw = json.load(f)
    mt = raw.get("model_type", "llama")
    if prefer_hf:
        try:
            if mt == "llama":
                from transformers import LlamaConfig as C
            elif mt == "gpt_neox":
                from transformers import GPTNeoXConfig as C
            else:
                raise NotImplementedError(f"Unknown model config type {mt}, only LLaMA and GPT-NeoX are supported")
            raw2 = {k: v for k, v in raw.items() if k not in ("architectures", "transformers_version")}
            return C(**raw2)
        except NotImplementedError:
            raise
        except Exception:
            pass
    return SimpleConfig(**raw)


def rope_settings(config):
    """(rotary fraction, base, scaling dict) from either config dialect: the classic GPT-NeoX fields ``rotary_pct`` /
    ``rotary_emb_base`` / ``rope_scaling`` (modeling_pythia.py:95-106 of the reference, checkpoints' ``config.json``; Llama has ``rope_theta``) or the
    ``rope_parameters`` dict that transformers >= 5 folds them into (``partial_rotary_factor``, ``rope_theta``, ``rope_type``, ``factor``)."""
    rp = getattr(config, "rope_parameters", None) or {}
    pct = getattr(config, "rotary_pct", None)
    if pct is None:
        pct = rp.get("partial_rotary_factor", getattr(config, "partial_rotary_factor", 0.25))
    base = getattr(config, "rotary_emb_base", None)
    if base is None:
        base = rp.get("rope_theta", getattr(config, "rope_theta", 10000))
    scaling = getattr(config, "rope_scaling", None)
    if (scaling is None or not scaling.get("type", scaling.get("rope_type"))) and rp.get("rope_type") not in (None, "default"):
        scaling = {"type": rp["rope_type"], "factor": rp.get("factor", 1.0)}
    return float(pct), base, scaling


def rope_scaling(config):
    """The rotary scaling dict as the config declares it, with every key it carries: ``rope_scaling`` when that names a type,
    else the ``rope_parameters`` of transformers >= 5 when its ``rope_type`` is not ``default``; None when rotary embeddings
    are unscaled."""
    scaling = getattr(config, "rope_scaling", None)
    if scaling and scaling.get("type", scaling.get("rope_type")):
        return scaling
    rp = getattr(config, "rope_parameters", None) or {}
    return rp if rp.get("rope_type") not in (None, "default") else None


def config_to_dict(config) -> Dict[str, Any]:
    if hasattr(config, "to_dict"):
        return config.to_dict()
    return dict(vars(config))


def save_config(config, directory: str) -> None:
    os.makedirs(directory, exist_ok=True)
    if hasattr(config, "save_pretrained"):
        try:
            config.save_pretrained(directory)
            return
        except Exception:
            pass
    with open(os.path.join(directory, "config.json"), "w") as f:
        json.dump(config_to_dict(config), f, indent=2, sort_keys=True, default=str)
