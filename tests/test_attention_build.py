"""Build-time facts of the attention kernels (no GPU): every head-size instantiation compiles without spills and fits the
H100's shared memory, and the routing rule for `--attention`."""
import importlib
import os
import re

import pytest

SMEM_PER_CTA = 227 * 1024  # H100: largest dynamic shared memory a CTA may opt into


def _attention_ptxas():
    """{(kernel, NP): {"regs", "spill_stores", "smem"}} from the -Xptxas -v log of the last build of attention.cu."""
    build = importlib.import_module("relora_b200.csrc.build")  # the package re-exports a build() function under that name
    if not os.path.exists(os.path.join(build.BUILD_DIR, "attention.cu.log")):
        pytest.skip("needs the built extension")
    out, cur = {}, None
    for line in build.ptxas_report().splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            k = re.search(r"(attn_[a-z_]+_kernel)(?:ILi(\d)E)?", m.group(1))
            cur = (k.group(1), int(k.group(2) or 0)) if k else None
            if cur:
                out[cur] = {"smem": 0}
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m:
            out[cur]["spill_stores"] = int(m.group(1))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out[cur]["regs"] = int(m.group(1))
            s = re.search(r"(\d+) bytes smem", line)
            out[cur]["smem"] = int(s.group(1)) if s else 0
    return out


def test_every_attention_instantiation_compiles_without_spills_and_fits_shared_memory():
    rows = _attention_ptxas()
    for kern in ("attn_fwd_kernel", "attn_bwd_dq_kernel", "attn_bwd_dkv_kernel"):
        assert {np for k, np in rows if k == kern} == {1, 2, 3, 4}, (kern, sorted(rows))
    import relora_b200._C as C

    for (kern, np_), r in rows.items():
        assert r["spill_stores"] == 0, (kern, np_, r)
        if np_:
            assert r["smem"] + C.attention_smem_bytes(64 * np_) <= SMEM_PER_CTA, (kern, np_, r)
    # head_dim <= 64 keeps the register budget of the single-panel kernels
    assert rows[("attn_fwd_kernel", 1)]["regs"] <= 90
    assert rows[("attn_bwd_dq_kernel", 1)]["regs"] <= 126
    assert rows[("attn_bwd_dkv_kernel", 1)]["regs"] <= 168


def test_attention_routing_rule():
    from relora_b200.ops.fused import attention_backend

    for hd in (16, 48, 64):
        assert [attention_backend(hd, m) for m in ("auto", "native", "sdpa")] == ["native", "native", "sdpa"]
    for hd in (80, 128, 256):
        assert [attention_backend(hd, m) for m in ("auto", "native", "sdpa")] == ["sdpa", "native", "sdpa"]
    for hd in (52, 84, 264, 512):
        assert [attention_backend(hd, m) for m in ("auto", "native", "sdpa")] == ["sdpa", "sdpa", "sdpa"]
    with pytest.raises(ValueError):
        attention_backend(64, "flash")


def test_attention_mode_comes_from_the_environment(monkeypatch):
    import torch

    from relora_b200.ops.fused import attention_backend

    monkeypatch.setenv("RELORA_B200_ATTENTION", "native")
    assert attention_backend(128) == "native"
    assert attention_backend(128, q=torch.zeros(1, 1, 1, 128, dtype=torch.bfloat16)) == "sdpa"  # CPU tensor
    monkeypatch.setenv("RELORA_B200_ATTENTION", "sdpa")
    assert attention_backend(64) == "sdpa"
    monkeypatch.delenv("RELORA_B200_ATTENTION")
    assert attention_backend(64) == "native" and attention_backend(128) == "sdpa"
