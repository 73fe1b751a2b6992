"""Edge cases the reference's tests exercise implicitly (directed test graphs with zero-degree nodes, None
weights, tiny graphs) plus ABI-level robustness: empty edge lists, N=1, non-contiguous inputs, B=0, inf norms."""
import pytest
import torch

from oracle import pyg, recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN, DCRNN, GConvGRU, GConvLSTM, TGCN
from pytorch_geometric_temporal_b200.plan import GraphPlan

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _close(got, want, rtol=1e-4, atol=1e-5):
    got = got.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol, equal_nan=True), f"max abs err {(got - want).abs().max():.3e}"


def test_empty_edge_list_all_flavors():
    ei = torch.zeros(2, 0, dtype=torch.long)
    x = torch.randn(6, 5)
    for flavor, kw in ((_lib.FLAVOR_CHEB, dict(normalization="sym")), (_lib.FLAVOR_GCN, {}), (_lib.FLAVOR_DCONV, {})):
        plan = GraphPlan(flavor, ei.to(DEV), None, 6, **kw)
        y = ops.spmm_raw(plan, 0, x.to(DEV)).cpu()
        if flavor == _lib.FLAVOR_GCN:      # only the added self loops remain: A^ = I
            assert torch.equal(y, x)
        elif flavor == _lib.FLAVOR_DCONV:
            assert torch.equal(y, torch.zeros_like(x))
    torch.manual_seed(0)
    m = GConvGRU(5, 8, 3)
    want = R.gconv_gru_cell(m.state_dict(), x, ei)
    _close(m.to(DEV)(x.to(DEV), ei.to(DEV)), want)


def test_single_node_and_tiny_graphs():
    ei = torch.tensor([[0], [0]])
    x = torch.randn(1, 3)
    torch.manual_seed(0)
    m = TGCN(3, 4)
    _close(m.to(DEV)(x.to(DEV), ei.to(DEV)), R.tgcn_cell(m.cpu().state_dict(), x, ei))
    m = DCRNN(3, 32, 2)   # N=1 through the fused wgmma kernel
    want = R.dcrnn_cell(m.state_dict(), x, ei)
    with torch.no_grad():
        _close(m.to(DEV)(x.to(DEV), ei.to(DEV)), want)


def test_zero_degree_nodes_propagate_inf_like_the_reference():
    """test/recurrent_test.py builds DIRECTED graphs: nodes without in-edges give 1/0 = inf norms (dcrnn.py:70-74);
    the reference output then holds inf/nan and its (shape-only) test still passes.  Same non-finite pattern here."""
    ei = torch.tensor([[0, 1, 2, 3], [1, 2, 3, 4]])   # path 0->1->2->3->4 : node 0 has no in-edge, node 4 no out-edge
    x, h = torch.randn(5, 2), torch.randn(5, 8)
    torch.manual_seed(0)
    m = DCRNN(2, 8, 2)
    want = R.dcrnn_cell(m.state_dict(), x, ei, None, h)
    got = m.to(DEV)(x.to(DEV), ei.to(DEV), None, h.to(DEV)).detach().cpu()
    assert got.shape == want.shape
    assert torch.equal(torch.isfinite(got), torch.isfinite(want))
    fin = torch.isfinite(want)
    assert torch.allclose(got[fin], want[fin], rtol=1e-4, atol=1e-5)


def test_non_contiguous_and_strided_inputs():
    g = torch.Generator().manual_seed(1)
    ei = torch.randint(0, 30, (2, 120), generator=g)
    ew = torch.rand(120, generator=g) + 0.1
    torch.manual_seed(0)
    m = GConvLSTM(6, 8, 2)
    Xbig, Hbig = torch.randn(30, 12), torch.randn(30, 16)
    X, H = Xbig[:, ::2], Hbig[:, 8:]          # strided views
    want = R.gconv_lstm_cell(m.state_dict(), X, ei, ew, H)
    got = m.to(DEV)(Xbig.to(DEV)[:, ::2], ei.to(DEV), ew.to(DEV), Hbig.to(DEV)[:, 8:])
    _close(got[0], want[0]); _close(got[1], want[1])
    eiT = ei.t().contiguous().to(DEV).t()     # non-contiguous [2,E] view
    got = m(Xbig.to(DEV)[:, ::2], eiT, ew.to(DEV), Hbig.to(DEV)[:, 8:])
    _close(got[0], want[0])


def test_zero_windows_and_zero_steps():
    ei = torch.tensor([[0, 1, 2], [1, 2, 0]], device=DEV)
    ew = torch.ones(3, device=DEV)
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    with torch.no_grad():
        assert m(torch.zeros(0, 12, 3, 2, device=DEV), ei, ew).shape == (0, 12, 3, 32)
        assert m(torch.zeros(4, 0, 3, 2, device=DEV), ei, ew).shape == (4, 0, 3, 32)


def test_plan_cache_tracks_in_place_edits():
    """Freshness by (data_ptr, _version): an in-place edit of edge_weight must rebuild the plan."""
    ei = torch.tensor([[0, 1, 2, 0], [1, 2, 0, 0]], device=DEV)
    ew = torch.tensor([1.0, 2.0, 3.0, 1.0], device=DEV)
    x, h = torch.randn(3, 2, device=DEV), torch.randn(3, 32, device=DEV)
    torch.manual_seed(0)
    m = DCRNN(2, 32, 2).to(DEV)
    with torch.no_grad():
        a = m(x, ei, ew, h)
        ew.mul_(torch.tensor([1.0, 5.0, 1.0, 1.0], device=DEV))
        b = m(x, ei, ew, h)
        want = R.dcrnn_cell({k: v.cpu() for k, v in m.state_dict().items()}, x.cpu(), ei.cpu(), ew.cpu(), h.cpu())
    assert not torch.allclose(a, b)
    _close(b, want)


def test_wrong_shapes_raise_runtime_errors():
    ei = torch.tensor([[0, 1], [1, 0]], device=DEV)
    m = DCRNN(2, 8, 2).to(DEV)
    with pytest.raises(RuntimeError):
        m(torch.randn(2, 3, device=DEV), ei)                      # wrong feature width
    with pytest.raises(RuntimeError, match="outside"):
        m(torch.randn(1, 2, device=DEV), ei)                      # edge_index refers to node 1 of a 1-node X
    plan = GraphPlan(_lib.FLAVOR_GCN, ei, None, 2)
    with pytest.raises(RuntimeError):
        ops.spmm_raw(plan, 0, torch.randn(3, 4, device=DEV))      # N mismatch
    with pytest.raises(ValueError):
        ops.spmm_raw(plan, 5, torch.randn(2, 4, device=DEV))      # operator index out of range
