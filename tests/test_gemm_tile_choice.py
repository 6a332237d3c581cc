"""Tile-width rule of the wgmma GEMM (no GPU): auto runs hidden-width bf16 outputs on 192-wide tiles where that takes fewer
tile-times on 132 SMs, and keeps 128 everywhere else.  Checked through gemm_plan, which runs the host-side schedule only."""
import pytest

from relora_b200.ops import native

SMEM_PER_BLOCK_OPTIN = 232448  # H100: largest dynamic shared memory one CTA may opt in to
SMS = 132                      # H100 SXM


@pytest.fixture(scope="module")
def plan():
    if not native.available():
        pytest.skip("needs the built extension")
    return native.module().gemm_plan


def _auto(plan, m, n, k, npg=0, out_f32=False, accumulate=False, split_k=1):
    return plan(0, out_f32, 4096, n, n, split_k, m=m, k=k, n_per_group=npg, accumulate=accumulate, sms=SMS)[0]


@pytest.mark.parametrize("n,k,npg", [
    (768, 768, 0),    # o forward, and the input gradients of q / k / v, o and gate / up with K 768 .. 2304
    (768, 2560, 0),   # down forward
    (768, 5120, 0),   # the gate / up input gradient's base product
    (2304, 768, 768),  # qkv forward: three groups of 768
])
def test_auto_is_192_for_hidden_width_outputs_of_llama_250m(plan, n, k, npg):
    assert _auto(plan, 12288, n, k, npg) == 192


@pytest.mark.parametrize("n,k,npg", [(5120, 768, 2560), (2560, 768, 0), (5120, 768, 0), (384, 768, 128)])
def test_auto_is_128_where_192_takes_as_long_or_longer_on_llama_250m(plan, n, k, npg):
    assert _auto(plan, 12288, n, k, npg) == 128


@pytest.mark.parametrize("n,k,npg", [
    (6144, 2048, 2048), (2048, 2048, 0), (11008, 2048, 5504), (2048, 5504, 0),  # forward
    (2048, 6144, 0), (2048, 11008, 0), (5504, 2048, 0),                        # input gradients
])
def test_auto_is_128_on_every_llama_1b_shape(plan, n, k, npg):
    assert _auto(plan, 8192, n, k, npg) == 128


def test_auto_is_128_for_fp32_accumulated_and_split_k_outputs(plan):
    assert _auto(plan, 12288, 768, 768, out_f32=True) == 128
    assert _auto(plan, 12288, 768, 768, out_f32=True, accumulate=True) == 128
    assert _auto(plan, 12288, 768, 768, accumulate=True) == 128
    assert _auto(plan, 12288, 768, 768, split_k=4) == 128


def test_auto_is_128_without_a_shape_or_a_device(plan):
    assert plan(0, False, 4096, 768, 768, 1)[0] == 128                   # M unknown
    assert plan(0, False, 4096, 768, 768, 1, m=12288, k=768, sms=0)[0] in (128, 192)  # this device's SMs, if any


def test_explicit_width_overrides_the_rule(plan):
    assert plan(128, False, 4096, 768, 768, 1, m=12288, k=768, sms=SMS)[0] == 128
    assert plan(192, False, 4096, 5120, 5120, 1, m=12288, k=768, sms=SMS)[0] == 192
    assert plan(256, False, 4096, 768, 768, 1, m=12288, k=768, sms=SMS)[0] == 256


def test_192_wide_tile_stores_through_tma_and_never_pairs(plan):
    bn, tma, smem, paired = plan(192, False, 4096, 768, 768, 1, m=12288, k=5120, pair=1, sms=SMS)
    assert (bn, tma, paired) == (192, True, False)
    # 4 stages of (16 + 24) KB, 2 KB of barriers / alignment, 48 KB of staging (2 warpgroups x 3 sub-tiles of 64 x 64)
    assert smem == 4 * 40 * 1024 + 2048 + 48 * 1024
    assert smem <= SMEM_PER_BLOCK_OPTIN
    assert plan(192, True, 4096, 768, 768, 1)[1] is False  # fp32 outputs keep the register epilogue
