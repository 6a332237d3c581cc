"""Build-time facts of the 192-wide tile (no GPU): the 128-wide GEMM kernels and the LoRA input-gradient kernel carry the
m64n192k16 wgmma of their 192-wide tiles, and the 256-wide GEMM kernels do not.  (test_wgmma_pipeline_build.py checks that
every one of these kernels issues its wgmma in batches and spills nothing.)"""
import collections
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n192_per_kernel():
    so = os.path.join(ROOT, "relora_b200", "_C.so")
    if shutil.which("cuobjdump") is None or not os.path.exists(so):
        pytest.skip("needs cuobjdump and the built extension")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    counts, fn = collections.Counter(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            counts[fn] += 0
        elif fn is not None and "HGMMA.64x192x16" in line:
            counts[fn] += 1
    return counts


def test_192_wide_wgmma_lives_in_the_128_wide_kernels():
    counts = _n192_per_kernel()
    gemm128 = [k for k in counts if k.startswith("_ZN2rb11gemm_kernelILi128E")]
    gemm256 = [k for k in counts if k.startswith("_ZN2rb11gemm_kernelILi256E")]
    lora_dx = [k for k in counts if k.startswith("_ZN2rb14lora_dx_kernel")]
    assert len(gemm128) == 4 and len(gemm256) == 4 and len(lora_dx) == 1, sorted(counts)
    assert all(counts[k] > 0 for k in gemm128 + lora_dx), {k: counts[k] for k in gemm128 + lora_dx}
    assert all(counts[k] == 0 for k in gemm256), {k: counts[k] for k in gemm256}
