"""Host side of BatchedDCRNN on the 64-wide row-split kernels (stmp_dcrnn_wide_rows_*): the routing of a call (`BatchedDCRNN._rows_ok`,
which checks the module's attributes before it consults the library), the autograd Function `_DcrnnHoistedRowsFn` and the hand-off of its
operands to `_weight_grads`, with every library call replaced by a dense torch restatement of its contract on the dense DConv
operators -- the output, gX and EVERY parameter gradient against the tiled path on the golden's models and graphs
(tests/golden/make_goldens_dcrnn_wide_rows.py: BatchedDCRNN(2, 64, 3) on the METR-LA shape and (2, 64, 2) on the PEMS-BAY shape)."""
import gzip
import importlib.util
import os
import types

import pytest
import torch

from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN
from test_dcrnn_narrow_rows_cpu import fake_hoisted_rows
from test_modules_host_logic_cpu import dense_dconv_gcn_ops  # noqa: F401  (dense DConv operators + SpMM, one-SM kernels off)


def _load(golden_dir, name):
    with gzip.open(os.path.join(golden_dir, f"dcrnn_wide_rows_{name}.pt.gz"), "rb") as f:
        g = torch.load(f, weights_only=False)
    spec = importlib.util.spec_from_file_location("_mk_wrows", os.path.join(golden_dir, "make_goldens_dcrnn_wide_rows.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g["edge_index"], g["edge_weight"], g["X"], g["K"] = mod.inputs(name)
    m = BatchedDCRNN(2, 64, g["K"])
    m.load_state_dict(mod.params([(n_, p.shape) for n_, p in m.named_parameters()], 11))
    return g, m


@pytest.fixture()
def dense_wrows(dense_dconv_gcn_ops, monkeypatch):   # noqa: F811
    return fake_hoisted_rows(monkeypatch, "stmp_dcrnn_wide_rows_supported")


def _close(got, want, rtol=1e-4, atol=1e-5):
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _grad_close(got, ref):
    _close(got, ref, 1e-3, 1e-3 * max(ref.abs().max().item(), 1e-12))


@pytest.mark.parametrize("name", ["metr_la", "pems_bay"])
def test_64_channels_route_to_the_hoisted_rows_path_and_match_the_tiled_path(golden_dir, dense_wrows, name):
    """The fused route (fakes) against the tiled path on the same dense operators: the output, gX and every parameter gradient, so the
    Function's hand-off to `_weight_grads` (layouts of S1 / S2 / dph / dpzr, the gradient order) is checked on the golden's shapes."""
    g, m = _load(golden_dir, name)
    ei, ew, X0 = g["edge_index"], g["edge_weight"], g["X"][:, :3]
    with torch.no_grad():
        m(X0, ei, ew)
    assert dense_wrows == ["fwd"]
    res = []
    for fused in (True, False):
        m._fused_training = fused
        m.zero_grad(set_to_none=True)
        X = X0.clone().requires_grad_(True)
        out = m(X, ei, ew)
        (out * torch.linspace(-1, 1, out.numel()).view_as(out)).sum().backward()
        res.append([out.detach(), X.grad] + [p.grad for p in m.parameters()])
    assert dense_wrows == ["fwd", "fwd", "bwd"]
    (of, *gf), (oa, *ga) = res
    _close(of, oa)
    for a, b in zip(gf, ga):
        _grad_close(a, b)


def test_hoisted_rows_no_bias_and_no_x_grad_bookkeeping(golden_dir, dense_wrows):
    """Without biases the Function returns no bias gradients; without an X gradient it asks the backward for no dX."""
    g, _ = _load(golden_dir, "metr_la")
    m = BatchedDCRNN(2, 64, 3, bias=False)
    out = m(g["X"][:, :2], g["edge_index"], g["edge_weight"])
    out.sum().backward()
    assert dense_wrows == ["fwd", "bwd"]
    assert all(p.grad is not None and p.grad.shape == p.shape for p in m.parameters())


def test_rows_ok_checks_the_envelope_before_the_plan(dense_wrows):
    """Shapes outside every row-split envelope are refused from the module's attributes alone: the plan is never consulted.  (2, 32, 2)
    is inside the 32-wide envelope; that it never reaches the 64-wide entry is checked by the fixture's library."""
    class NoPlan:
        def __getattr__(self, k):
            raise AssertionError("plan consulted")
    X = torch.zeros(1, 1, 3, 2)
    for cin, cout, K in ((2, 64, 1), (2, 64, 4), (5, 64, 2), (2, 16, 3)):
        assert not BatchedDCRNN(cin, cout, K)._rows_ok(NoPlan(), X, False)
    assert not BatchedDCRNN(2, 64, 3)._rows_ok(NoPlan(), X.double(), False)
    m = BatchedDCRNN(2, 64, 3)
    m._fused_training = False
    assert not m._rows_ok(NoPlan(), X, True)
    with pytest.raises(pytest.fail.Exception, match="stmp_dcrnn_rows_supported consulted"):
        BatchedDCRNN(2, 32, 2)._rows_ok(types.SimpleNamespace(handle=None), X, False)


def test_wide_fused_training_off_and_shapes_outside_the_envelope_keep_the_tiled_path(golden_dir, dense_wrows):
    g, m = _load(golden_dir, "metr_la")
    X = g["X"][:, :2]
    m._fused_training = False
    m(X.clone().requires_grad_(True), g["edge_index"], g["edge_weight"]).sum().backward()
    assert dense_wrows == ["fwd"] or dense_wrows == []
    dense_wrows.clear()
    for cin, K in ((2, 1), (2, 4), (5, 2)):
        mm = BatchedDCRNN(cin, 64, K)
        with torch.no_grad():
            mm(torch.randn(1, 2, 207, cin), g["edge_index"], g["edge_weight"])
    assert dense_wrows == []
