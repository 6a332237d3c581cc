"""Host-side pairing rule of the wgmma GEMM and the LoRA input-gradient kernel (no GPU), and lora_dx's epilogue choice."""
import pytest

from relora_b200.ops import native


@pytest.fixture(scope="module")
def C():
    if not native.available():
        pytest.skip("needs the built extension")
    return native.module()


def _paired(C, block_n=0, m=12288, n=2048, k=2048, m_per_group=0, pair=-1):
    return C.gemm_plan(block_n, False, 4096, n, n, 1, m=m, m_per_group=m_per_group, pair=pair, k=k)[3]


def test_auto_pairs_long_reductions_into_wide_outputs(C):
    assert _paired(C) and _paired(C, block_n=128) and _paired(C, n=11008, k=2048) and _paired(C, n=2048, k=5504)
    assert _paired(C, m=12416) and _paired(C, m=129)  # odd tile counts: the last pair's second tile lies past M
    # measured slower or no faster: N 768 (any K), K 768 (any N)
    assert not _paired(C, n=768, k=5120) and not _paired(C, n=5120, k=768) and not _paired(C, n=2304, k=768)
    assert _paired(C, n=768, k=768, pair=1)  # on request wherever the form allows


def test_pairing_is_off_where_the_form_does_not_allow_it(C):
    assert not _paired(C, pair=0)
    assert not _paired(C, block_n=256) and not _paired(C, block_n=256, pair=1)  # the 256-wide tile ignores the request
    assert not _paired(C, m=128) and not _paired(C, m=1)  # a single M tile
    # M groups of the weight gradients: a pair shares one B tile, so a group must hold whole pairs
    assert not _paired(C, m=384, m_per_group=128) and not _paired(C, m=1152, m_per_group=384)
    assert _paired(C, m=768, m_per_group=256) and _paired(C, m=1024, m_per_group=512)


def test_plan_keeps_its_first_fields(C):
    assert C.gemm_plan(0, False, 4096, 5120, 5120, 1)[:3] == C.gemm_plan(0, False, 4096, 5120, 5120, 1, m=12288)[:3]


@pytest.mark.parametrize("m,n,kb,pair,expect", [
    (8192, 5504, 2048, -1, (True, True)), (8192, 2048, 2048, -1, (True, True)), (8192, 2048, 2048, 0, (False, True)),
    (12288, 768, 2304, -1, (False, True)), (12288, 2560, 768, -1, (False, True)), (128, 5504, 2048, 1, (False, True)),
    (329, 1000, 0, 1, (True, True)), (329, 1002, 0, 1, (True, False)),  # a row of 1002 bf16 ends in half a 16-byte chunk
])
def test_lora_dx_plan(C, m, n, kb, pair, expect):
    assert C.lora_dx_plan(m, n, pair, kb=kb) == expect
