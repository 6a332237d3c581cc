"""Build-time facts of the wgmma kernels (no GPU): ptxas issues their wgmma in batches rather than one at a time.

ptxas serialises every wgmma of a kernel (each one waits for the previous to finish) when a function call sits on a path
the wgmma pipeline crosses (warning C7510), and it serialises single wgmma that are issued under a condition of their own
or whose operand registers are written inside a batch.  In the SASS a serialised wgmma carries its own ``gsb0`` and is
followed by a wait; a batch of them carries one ``gsb0``, on its last instruction.
"""
import importlib
import os
import re
import shutil

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOT = ("gemm_kernel<", "lora_dx_kernel", "attn_fwd_kernel<", "attn_bwd_dq_kernel<", "attn_bwd_dkv_kernel<")


def _ptxas_log():
    build = importlib.import_module("relora_b200.csrc.build")
    if not os.path.exists(os.path.join(build.BUILD_DIR, "gemm_wgmma.cu.log")):
        pytest.skip("needs the built extension")
    return build.ptxas_report()


def _census():
    so = os.path.join(ROOT, "relora_b200", "_C.so")
    if shutil.which("cuobjdump") is None or not os.path.exists(so):
        pytest.skip("needs cuobjdump and the built extension")
    from tools import sass_census

    return sass_census.census(so)


def test_no_wgmma_pipeline_crosses_a_function_call():
    log = _ptxas_log()
    assert "C7510" not in log, [ln for ln in log.splitlines() if "C7510" in ln][:3]


def test_wgmma_kernels_do_not_spill():
    spills, cur = {}, None
    for line in _ptxas_log().splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None and re.search(r"gemm_kernel|lora_dx_kernel|attn_(fwd|bwd_dq|bwd_dkv)_kernel", cur):
            spills[cur] = int(m.group(1)) + int(m.group(2))
    assert len(spills) >= 8 + 1 + 12, sorted(spills)
    assert all(v == 0 for v in spills.values()), {k: v for k, v in spills.items() if v}


def test_gemm_and_attention_issue_wgmma_in_batches():
    rows = {k: c for k, c in _census().items() if k.startswith(HOT)}
    assert sum(k.startswith("gemm_kernel<") for k in rows) == 8, sorted(rows)
    assert sum(k.startswith("attn_") for k in rows) == 12, sorted(rows)
    assert "lora_dx_kernel" in rows
    for k, c in rows.items():
        gmma = c["HGMMA"] + c["QGMMA"]
        # GEMM: one k-block of 4 wgmma per batch.  Attention: each product is a batch of >= 4 wgmma.
        assert gmma > 0 and 4 * c["gsb0"] <= gmma, (k, dict(c))
