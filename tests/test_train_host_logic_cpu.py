"""Host side of the training-path additions, no GPU: the run-time switches the tests' reference paths sit behind are accepted by the
C ABI (and unknown or retired names rejected), the flat optimizer refuses to run without CUDA (no CPU fallback), the basis row pitch helper, and
the differentiable weight folding of the TGCN family equals the cached inference packing."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, distributed as D, ops
from pytorch_geometric_temporal_b200.nn.recurrent import TGCN


def test_only_the_reference_path_switches_are_known_to_the_library():
    for name in ("dcrnn_tc", "dcrnn_fwd_split", "dcrnn_bwd_split", "dcrnn_wgrad_tc"):
        _lib.set_option(name, 1)                           # host-only: no CUDA call behind it
    for name in ("no_such_switch", "spmm_variant", "spmm_block", "spmm_rows_per_group", "dcrnn_bwd_all_cin"):
        with pytest.raises(ValueError):
            _lib.set_option(name, 1)


def test_flat_adam_has_no_cpu_fallback():
    m = torch.nn.Linear(3, 2)
    sync = D.FlatGradSync(m.parameters())
    with pytest.raises(RuntimeError):
        D.FlatAdam(sync)
    # the gradient views survive and still alias the flat buffer
    m(torch.ones(1, 3)).sum().backward()
    assert float(sync.flat.abs().sum()) > 0
    assert all(p.grad.data_ptr() >= sync.flat.data_ptr() for p in m.parameters())


def test_basis_row_pitch_is_whole_sectors():
    for cin in (1, 2, 3, 4):
        ld = ops.dcrnn_bwd_basis_ld(cin, 32, 2)
        assert ld % 8 == 0 and 3 * (cin + 32) <= ld < 3 * (cin + 32) + 8


@pytest.mark.parametrize("cin", [1, 2, 4])
def test_tgcn_differentiable_folding_equals_the_cached_packing(cin):
    torch.manual_seed(cin)
    m = TGCN(cin, 32)
    for p in m.parameters():
        torch.nn.init.normal_(p, std=0.3)
    A, Bm, c = m._fold3()
    with torch.no_grad():
        A0, B0, c0 = m._packed3()
    assert torch.equal(A.detach(), A0) and torch.equal(Bm.detach(), B0) and torch.equal(c.detach(), c0)
    # gradients reach every parameter the folded matrices depend on (the r gate only through A / c / Bm)
    (A.square().sum() + Bm.square().sum() + c.square().sum()).backward()
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())
