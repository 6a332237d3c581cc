"""cross_entropy_fwd_bwd past the shared-memory staging limit (H100: -m gpu): vocabularies above 102,400 take the streaming kernel,
checked element by element against ops.reference.cross_entropy_ref, with a row pitch wider than V whose extra columns must stay
untouched, ignored rows, labels 0 and V - 1, a gradient scale, accumulators that start non-zero and logits spread over a wide
range.  At V = 102,400 the call still takes the single-pass kernel."""
import math

import pytest
import torch

from guarded_buffers import Guarded
from relora_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


@pytest.fixture(scope="module")
def C():
    from relora_b200.ops import native

    return native.require()


def _logits(M, V, g):
    """Rows of N(0, σ²) with σ from 0.5 to 16, offsets in [-60, 60] and one spike of +30 in every third row."""
    x = torch.randn(M, V, generator=g) * torch.logspace(math.log10(0.5), math.log10(16.0), M).view(M, 1)
    x += torch.empty(M, 1).uniform_(-60, 60, generator=g)
    rows = torch.arange(0, M, 3)
    x[rows, torch.randint(0, V, (rows.numel(),), generator=g)] += 30.0
    return x.to(BF)


def _labels(M, V, g, ignore_index=-100):
    y = torch.randint(0, V, (M,), generator=g)
    y[0], y[1], y[2] = 0, V - 1, ignore_index
    y[M // 2] = ignore_index
    return y


def _check(C, logits, labels, V, grad_scale, ld_view):
    """Runs the kernel on ``ld_view`` (the logits at their pitch, as the binding receives them) and checks every output."""
    before = logits.clone()
    loss0 = torch.tensor([2.5], device="cuda")
    count0 = torch.tensor([3.0], device="cuda")
    loss_sum, count = loss0.clone(), count0.clone()
    C.cross_entropy_fwd_bwd(ld_view, labels, V, grad_scale, -100, loss_sum, count)
    torch.cuda.synchronize()
    r = ref.cross_entropy_ref(before, labels, V, grad_scale, -100, loss0, count0)
    ref.assert_rowwise_close("ce grad", logits[:, :V], *r["grad"])
    ref.assert_rowwise_close("ce loss_sum", loss_sum, *r["loss_sum"])
    ref.assert_bitwise_equal("ce count", count, r["count"].to(torch.float32))
    ignored = labels == -100
    assert bool((logits[ignored, :V].float() == 0).all()), "ignored rows must be exact zeros"
    assert bool((logits[~ignored, :V].float() != 0).any())


@pytest.mark.parametrize("V", [102401, 128256, 131077, 256000])
@pytest.mark.parametrize("grad_scale", [1.0, 0.37])
def test_streaming_cross_entropy_matches_the_reference(C, V, grad_scale):
    """Operand inside a NaN guard (a read past V or past the last row poisons a row's max); the guard must survive bit for bit."""
    g = torch.Generator().manual_seed(V)
    M = 41
    x = _logits(M, V, g)
    labels = _labels(M, V, g).cuda()
    buf = Guarded(x.cuda(), float("nan"))
    assert buf.view.stride(0) > V
    _check(C, buf.view, labels, V, grad_scale, buf.view)
    assert buf.guards_intact(), "the kernel wrote outside the [M, V] logits"


@pytest.mark.parametrize("V", [128256, 131077])
def test_padding_columns_of_the_executor_layout_stay_untouched(C, V):
    """The fused executors' layout: a [M, ldv] chunk with V < ldv, the columns [V, ldv) holding canaries."""
    g = torch.Generator().manual_seed(1)
    M, ldv = 23, (V + 7) // 8 * 8 + 8
    lg = torch.full((M, ldv), 1234.0, dtype=BF)
    lg[:, :V] = _logits(M, V, g)
    lg = lg.cuda()
    labels = _labels(M, V, g).cuda()
    canary = lg[:, V:].clone()
    _check(C, lg, labels, V, 0.5, lg)
    ref.assert_bitwise_equal("ce padding columns", lg[:, V:], canary)


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "ce_" in e.name and "kernel" in e.name]


def test_the_staging_limit_picks_the_kernel(C):
    """V = 102,400 (204,800 bytes a row) is the longest row the single-pass kernel stages; one more column streams."""
    names = {}
    for V in (102400, 102401):
        g = torch.Generator().manual_seed(V)
        lg = torch.zeros(8, (V + 7) // 8 * 8, dtype=BF)  # the row pitch the binding needs: a multiple of 16 bytes
        lg[:, :V] = _logits(8, V, g)
        lg = lg.cuda()
        labels = _labels(8, V, g).cuda()
        loss_sum = torch.zeros(1, device="cuda")
        count = torch.zeros(1, device="cuda")
        before = lg.clone()
        names[V] = _kernel_names(lambda: C.cross_entropy_fwd_bwd(lg, labels, V, 1.0, -100, loss_sum, count))
        r = ref.cross_entropy_ref(before, labels, V, 1.0, -100, torch.zeros(1), torch.zeros(1))
        ref.assert_rowwise_close(f"ce grad V={V}", lg[:, :V], *r["grad"])
    assert len(names[102400]) == 1 and "ce_kernel" in names[102400][0], names
    assert len(names[102401]) == 1 and "ce_stream_kernel" in names[102401][0], names
