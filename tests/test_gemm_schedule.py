"""Host-side schedule of the wgmma GEMM (no GPU): tile width, which outputs take the TMA-store epilogue, and the shared
memory each tile width asks for."""
import pytest

from relora_b200.ops import native

SMEM_PER_BLOCK_OPTIN = 232448  # H100: largest dynamic shared memory one CTA may opt in to


@pytest.fixture(scope="module")
def plan():
    if not native.available():
        pytest.skip("needs the built extension")
    return native.module().gemm_plan


def test_auto_tile_width_is_128(plan):
    assert plan(0, False, 4096, 5120, 5120, 1)[0] == 128
    assert plan(128, False, 4096, 5120, 5120, 1)[0] == 128
    assert plan(256, False, 4096, 5120, 5120, 1)[0] == 256


def test_shared_memory_budget(plan):
    smem128, smem256 = plan(128, False, 4096, 768, 768, 1)[2], plan(256, False, 4096, 768, 768, 1)[2]
    assert smem128 <= SMEM_PER_BLOCK_OPTIN and smem256 <= SMEM_PER_BLOCK_OPTIN
    # 6 stages of (16 + 16) KB and 4 of (16 + 32) KB, 2 KB of barriers / alignment; the 128-wide tile adds 32 KB of staging
    assert smem256 == 4 * 48 * 1024 + 2048
    assert smem128 == 6 * 32 * 1024 + 2048 + 32 * 1024


@pytest.mark.parametrize(
    "block_n, out_f32, addr, ldc, n, split_k, expect",
    [
        (0, False, 4096, 5120, 5120, 1, True),      # bf16 output, 16-byte aligned base, pitch and row length
        (0, False, 4096 + 32, 1072, 768, 1, True),  # column window of a wider buffer: still aligned
        (0, True, 4096, 5120, 5120, 1, False),      # fp32 output (weight gradients) keeps the register epilogue
        (0, True, 4096, 768, 768, 4, False),        # split-K partial sums go through atomics
        (0, False, 4096 + 2, 5120, 5120, 1, False),  # base not 16-byte aligned
        (0, False, 4096, 5121, 5120, 1, False),     # row pitch not a multiple of 16 bytes
        (0, False, 4096, 1072, 1001, 1, False),     # ragged last 16-byte chunk of a row (the store would pass column N)
        (0, False, 4096, 32104, 32100, 1, False),   # the LM head's vocabulary width
        (256, False, 4096, 5120, 5120, 1, False),   # the 256-wide tile stores from registers
    ],
)
def test_tma_store_choice(plan, block_n, out_f32, addr, ldc, n, split_k, expect):
    assert plan(block_n, out_f32, addr, ldc, n, split_k)[1] is expect
