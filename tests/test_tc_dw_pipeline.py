"""What the producer/consumer pipeline of tc_dw.cu can get wrong and test_tc_gemm.py::test_tc_dw (values
against float64) does not show: results that depend on timing, and writes outside the outputs.

M = 132*32*13 + 5 gives every CTA a slab of 14 chunks, several times the deepest shared-memory ring (4
stages), so every stage is refilled and both mbarrier phases of every stage are waited on more than once."""
import pytest
import torch

from test_tc_gemm import DW_SHAPES, SENTINEL, check, dev, gen, padded, randn, ref_affine  # noqa: F401

LONG_SLABS = 132 * 32 * 13 + 5


@pytest.mark.gpu
@pytest.mark.parametrize("co,ci", DW_SHAPES)
def test_tc_dw_is_deterministic(dev, gen, co, ci):
    """Two calls on the same inputs give bitwise the same dW, and it is the right one."""
    from superpoint_graph_b200 import ops
    M = LONG_SLABS
    dY, P = randn(gen, M, co), randn(gen, M, ci) * 1.3 + 0.2
    scale, shift = torch.rand(ci, generator=gen) + 0.5, randn(gen, ci)
    dYd, Pd, aff = dY.to(dev), P.to(dev), (scale.to(dev), shift.to(dev), True)
    first = ops.tc_dw(dYd, co, Pd, ci, M, co, ci, p_aff=aff).clone()
    second = ops.tc_dw(dYd, co, Pd, ci, M, co, ci, p_aff=aff)
    assert torch.equal(first, second)
    check("dw_long", first, dY.double().t() @ ref_affine(P.double(), scale.double(), shift.double(), True), 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("co,ci", [(64, 32), (128, 128), (256, 128)])
def test_tc_dw_write_set(dev, gen, co, ci):
    """Through the C-ABI with sentinel-filled slack behind the workspace and behind dW: the call writes
    ctas*co*ci floats of workspace and the [co, ci] result, nothing else, and reads no padding column
    (NaN) and no row >= M of its operands."""
    from superpoint_graph_b200 import _lib, ops
    M, lddy, ldp, slack = LONG_SLABS, co + 4, ci + 8, 4096
    dY, P, shift = randn(gen, M, co), randn(gen, M, ci), randn(gen, ci)
    nan_rows = torch.full((32, max(lddy, ldp)), float("nan"))
    dYd = torch.cat([padded(dY, lddy), nan_rows[:, :lddy]]).to(dev)
    Pd = torch.cat([padded(P, ldp), nan_rows[:, :ldp]]).to(dev)
    shift_d = shift.to(dev)
    want = ops.tc_dw(dYd, lddy, Pd, ldp, M, co, ci, p_aff=(None, shift_d, False)).clone()
    used = int(_lib.lib().spg_tc_dw_ctas(M)) * co * ci
    ws = torch.full((used + slack,), SENTINEL, device=dev)
    dW = torch.full((co * ci + slack,), SENTINEL, device=dev)
    _lib.call("spg_tc_dw", dYd, lddy, Pd, ldp, None, shift_d, 0, dW, ws, M, co, ci, _lib.current_stream())
    assert torch.equal(dW[:co * ci].view(co, ci), want)
    assert bool((dW[co * ci:] == SENTINEL).all()) and bool((ws[used:] == SENTINEL).all())
    assert bool(torch.isfinite(ws[:used]).all())
