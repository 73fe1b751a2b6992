"""DyGrEncoder without a GPU: the float64 GatedGraphConv oracle against dense per-aggregation restatements and the reference's stored
results, the module's parameter layout and seeded init against the reference's, the routing predicate, and the errors the module and the
reference raise."""
import os
import sys

import pytest
import torch

from dygrae_seq import GatedGraphConv, aggregate, check_reference, load, oracle_run, states_for
from gconvgru_seq import chickenpox_train_split
from oracle import refload
from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import DyGrEncoder
from wikimaths_seq import load as load_wikimaths

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
D = torch.float64


def _reference_cls():
    sys.path.insert(0, refload._STUBS)
    import torch_geometric.nn as tgnn
    tgnn.GatedGraphConv = GatedGraphConv
    return refload.load("nn.recurrent.dygrae").DyGrEncoder


def test_aggregation_against_dense_loops():
    g = torch.Generator().manual_seed(5)
    ei = torch.tensor([[0, 1, 2, 2, 3, 4, 4, 5, 0, 7, 7], [1, 1, 0, 0, 5, 4, 2, 3, 6, 6, 6]])   # self loops, duplicates, isolated 8
    w = torch.tensor([1.0, -2.0, 0.5, 0.5, 0.0, 3.0, -1.0, 2.0, 1.5, 1.0, 1.0], dtype=D)
    m = torch.randn(9, 3, generator=g, dtype=D)
    for aggr in ("add", "mean", "max"):
        got = aggregate(m, ei, w, aggr)
        for i in range(9):
            msgs = [w[k] * m[ei[0, k]] for k in range(ei.size(1)) if ei[1, k] == i]
            if not msgs:
                want = torch.zeros(3, dtype=D)
            elif aggr == "max":
                want = torch.stack(msgs).max(0).values
            else:
                want = torch.stack(msgs).sum(0) / (len(msgs) if aggr == "mean" else 1)
            torch.testing.assert_close(got[i], want, rtol=1e-14, atol=1e-14)


def test_max_splits_tied_gradients_evenly():
    """Node 6 receives two identical messages from node 7 (a duplicate edge): each gets half of the gradient; a maximum of exactly 0
    counts the zero-initialised output as one more tie."""
    ei = torch.tensor([[7, 7, 1, 2], [6, 6, 0, 0]])
    m = torch.zeros(8, 1, dtype=D)
    m[7, 0], m[1, 0], m[2, 0] = 2.0, 0.0, -1.0
    m.requires_grad_(True)
    aggregate(m, ei, None, "max").sum().backward()
    assert m.grad[7, 0] == 1.0 and m.grad[1, 0] == 0.5 and m.grad[2, 0] == 0.0


def _graph(c):
    if c["graph"] == "chickenpox":
        return chickenpox_train_split()
    w = load_wikimaths(GOLDEN)
    return w["edge_index"], w["edge_weight"], w["X"], w["Y"]


@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_oracle_matches_reference(name):
    c = load(GOLDEN)["cases"][name]
    ei, ew, X, Y = _graph(c)
    H0, C0 = states_for(c, X.shape[1], dtype=D)
    outs, cost, leaves = oracle_run(c, X, Y, ei, ew, H0, C0)
    cost.backward()
    check_reference(c, outs.detach(), cost, {k: v.grad for k, v in leaves.items()},
                    None if H0 is None else H0.grad, None if C0 is None else C0.grad)


KEYS = ["conv_layer.weight", "conv_layer.rnn.weight_ih", "conv_layer.rnn.weight_hh", "conv_layer.rnn.bias_ih", "conv_layer.rnn.bias_hh"]


@pytest.mark.parametrize("C,Lg,aggr,Ho,Ll", [(4, 1, "mean", 32, 1), (16, 3, "max", 64, 2), (32, 2, "add", 7, 3)])
def test_state_dict_and_seeded_init_match_reference(C, Lg, aggr, Ho, Ll):
    ours = DyGrEncoder(C, Lg, aggr, Ho, Ll)
    lstm = [f"recurrent_layer.{p}_l{k}" for k in range(Ll) for p in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    assert list(ours.state_dict()) == KEYS + lstm
    assert ours.conv_layer.weight.shape == (Lg, C, C) and ours.conv_layer.rnn.weight_ih.shape == (3 * C, C)
    assert isinstance(ours.recurrent_layer, torch.nn.LSTM)
    if not refload.available():
        pytest.skip("reference tree not present")
    ref_cls = _reference_cls()
    torch.manual_seed(11)
    ref = ref_cls(C, Lg, aggr, Ho, Ll)
    torch.manual_seed(11)
    ours = DyGrEncoder(C, Lg, aggr, Ho, Ll)
    assert list(ref.state_dict()) == list(ours.state_dict())
    for k, v in ref.state_dict().items():
        assert torch.equal(v, ours.state_dict()[k]), k


def test_seeded_init_follows_pyg_draw_order():
    """GRUCell constructor draws, then U(-1/sqrt(C), 1/sqrt(C)) for weight, then the GRUCell's reset: replayed by hand."""
    torch.manual_seed(3)
    m = GatedGraphConv(5, 2, "add")
    torch.manual_seed(3)
    torch.nn.GRUCell(5, 5)
    w = torch.empty(2, 5, 5).uniform_(-5 ** -0.5, 5 ** -0.5)
    rnn = torch.nn.GRUCell(5, 5)            # same draws as rnn.reset_parameters(): four U(-1/sqrt(5), 1/sqrt(5)) tensors in order
    assert torch.equal(m.weight, w)
    for k, v in rnn.state_dict().items():
        assert torch.equal(getattr(m.rnn, k), v), k


def test_errors():
    with pytest.raises(AssertionError, match="Wrong aggregator."):
        DyGrEncoder(4, 1, "sum", 32, 1)
    m = DyGrEncoder(4, 1, "mean", 32, 1)
    ei = torch.tensor([[0, 1], [1, 0]])
    with pytest.raises(ValueError, match="input channels"):
        m(torch.zeros(2, 5), ei)
    with pytest.raises(ValueError, match="Invalid hidden state and cell matrices."):
        m(torch.zeros(2, 4), ei, None, torch.zeros(2, 32), None)
    with pytest.raises(ValueError, match="Invalid hidden state and cell matrices."):
        m(torch.zeros(2, 4), ei, None, None, torch.zeros(2, 32))


def test_carried_state_errors_of_the_reference():
    """The reference squeezes H and C: at N = 1 they come back as (H_h,) and feeding them back raises IndexError; with two LSTM layers
    they come back as (2, N, H_h), H[None] is 4-D and torch.nn.LSTM raises RuntimeError.  The module follows the same code there."""
    if not refload.available():
        pytest.skip("reference tree not present")
    ref_cls = _reference_cls()
    torch.manual_seed(0)
    m = ref_cls(4, 1, "mean", 32, 1)
    x, ei = torch.randn(1, 3), torch.zeros(2, 0, dtype=torch.int64)
    _, H, C = m(x, ei)
    assert H.shape == (32,)
    with pytest.raises(IndexError):
        m(x, ei, None, H, C)
    m = ref_cls(4, 1, "mean", 32, 2)
    x, ei = torch.randn(5, 3), torch.tensor([[0, 1], [1, 2]])
    _, H, C = m(x, ei)
    assert H.shape == (2, 5, 32)
    with pytest.raises(RuntimeError):
        m(x, ei, None, H, C)


class _Plan:
    num_nodes = 20


@pytest.mark.parametrize("F,C,dtype,ew,training,fused,want", [
    (4, 4, torch.float32, None, False, True, True), (1, 32, torch.float32, "f32", True, True, True),
    (32, 32, torch.float32, None, True, True, True), (5, 4, torch.float32, None, False, True, False),
    (4, 33, torch.float32, None, False, True, False), (4, 4, torch.float64, None, False, True, False),
    (4, 4, torch.float32, "f64", False, True, False), (4, 4, torch.float32, "grad", True, True, False),
    (4, 4, torch.float32, None, True, False, False), (4, 4, torch.float32, None, False, False, True)])
def test_conv_routing_predicate(F, C, dtype, ew, training, fused, want):
    m = DyGrEncoder(C, 2, "max", 32, 1)
    m.fused_training = fused
    X = torch.zeros(20, F, dtype=dtype)
    w = {None: None, "f32": torch.ones(7), "f64": torch.ones(7, dtype=torch.float64), "grad": torch.ones(7, requires_grad=True)}[ew]
    assert m._conv_ok(X, w, training) is want
    assert m._conv_ok(X.unsqueeze(0), None, training) is False


@pytest.mark.parametrize("F,C,Lg,training,fused,want", [
    (4, 4, 1, False, True, True), (4, 4, 1024, False, True, True), (4, 4, 1025, False, True, False), (4, 4, 1025, True, True, False),
    (1, 32, 2, True, True, True), (5, 4, 2, False, True, False), (4, 4, 2, True, False, False)])
def test_conv_route_asks_the_library(monkeypatch, F, C, Lg, training, fused, want):
    """_conv_route: the module's own conditions (_conv_ok), then the library's envelope, asked through ops.ggc_rows_supported and
    restated here (1 024 layers at most) so the route runs without the library.  The library is asked exactly when the module's
    conditions hold, with the plan, L_g, in_channels and C."""
    asked = []

    def supported(plan, num_layers, cin, channels):
        asked.append((plan, num_layers, cin, channels))
        return 1 <= num_layers <= 1024 and 1 <= cin <= channels <= 32
    monkeypatch.setattr(ops, "ggc_rows_supported", supported)
    m = DyGrEncoder(C, Lg, "add", 32, 1)
    m.fused_training = fused
    X = torch.zeros(20, F)
    plan = _Plan()
    assert m._conv_route(plan, X, None, training) is want
    assert asked == ([(plan, Lg, F, C)] if m._conv_ok(X, None, training) else [])


@pytest.mark.parametrize("C,Ho,Ll,shape,dtype,want", [
    (4, 32, 1, None, torch.float32, True), (16, 64, 1, (20, 64), torch.float32, True), (17, 32, 1, None, torch.float32, False),
    (4, 48, 1, None, torch.float32, False), (4, 32, 2, None, torch.float32, False), (4, 32, 1, (32,), torch.float32, False),
    (4, 32, 1, (20, 32), torch.float64, False)])
def test_lstm_routing_predicate(monkeypatch, C, Ho, Ll, shape, dtype, want):
    monkeypatch.setattr(ops, "lstm_rows_supported", lambda plan, variant, n_ops, c, o: n_ops == 0 and c <= 16 and o in (32, 64))
    m = DyGrEncoder(C, 1, "add", Ho, Ll)
    H = None if shape is None else torch.zeros(shape, dtype=dtype)
    assert m._lstm_ok(_Plan(), 20, H, None if H is None else H.clone()) is want
