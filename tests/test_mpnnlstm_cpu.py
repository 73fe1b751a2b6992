"""MPNNLSTM without a GPU: the float64 restatement against the reference's stored results, the state_dict keys and seeded initialisation
against the reference's, the reference's errors (a bad view, one row in training mode) and the routing predicate."""
import os

import pytest
import torch

from mpnnlstm_seq import Masks, check_reference, graph_of, load, oracle_run, reference_class
from oracle import refload
from pytorch_geometric_temporal_b200.nn.recurrent import MPNNLSTM

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_oracle_matches_reference(name):
    c = load(GOLDEN)["cases"][name]
    ei, ew, train, ev = graph_of(c, GOLDEN)
    outs, cost, evs, leaves, bufs = oracle_run(c, train, ev, ei, ew, c["epochs"])
    check_reference(c, outs.detach(), cost, evs, {k: v.grad for k, v in leaves.items()}, bufs)


KEYS = (["_convolution_1.bias", "_convolution_1.lin.weight", "_convolution_2.bias", "_convolution_2.lin.weight"]
        + [f"_batch_norm_{i}.{k}" for i in (1, 2) for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]
        + [f"_recurrent_{i}.{k}_l0" for i in (1, 2) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")])


@pytest.mark.parametrize("args", [(4, 32, 20, 1, 0.5), (64, 32, 100, 1, 0.5), (1, 32, 20, 4, 0.0), (14, 64, 1068, 2, 0.3)])
def test_state_dict_and_seeded_init_match_reference(args):
    ours = MPNNLSTM(*args)
    assert list(ours.state_dict()) == KEYS
    assert isinstance(ours._batch_norm_1, torch.nn.BatchNorm1d) and isinstance(ours._recurrent_1, torch.nn.LSTM)
    assert (ours.in_channels, ours.hidden_size, ours.num_nodes, ours.window, ours.dropout) == args
    if not refload.available():
        pytest.skip("reference tree not present")
    torch.manual_seed(11)
    ref = reference_class(Masks(0))(*args)
    torch.manual_seed(11)
    ours = MPNNLSTM(*args)
    assert list(ref.state_dict()) == list(ours.state_dict())
    for k, v in ref.state_dict().items():
        assert torch.equal(v, ours.state_dict()[k]), k


@pytest.mark.parametrize("rows,window,nodes", [(30, 1, 20), (60, 4, 20), (7, 2, 3)])
def test_bad_view_raises_as_reference(rows, window, nodes):
    X, ei = torch.randn(rows, 4), torch.zeros(2, 0, dtype=torch.int64)
    with pytest.raises(RuntimeError) as ours:
        MPNNLSTM(4, 32, nodes, window, 0.5)(X, ei, None)
    if refload.available():
        with pytest.raises(RuntimeError) as ref:
            reference_class(Masks(0))(4, 32, nodes, window, 0.5)(X, ei, None)
        assert str(ours.value) == str(ref.value)


def test_one_row_in_training_raises_as_reference():
    X, ei = torch.randn(1, 4), torch.zeros(2, 0, dtype=torch.int64)
    with pytest.raises(ValueError) as ours:
        MPNNLSTM(4, 32, 1, 1, 0.5)(X, ei, None)
    assert str(ours.value) == "Expected more than 1 value per channel when training, got input size torch.Size([1, 32])"
    if refload.available():
        with pytest.raises(ValueError) as ref:
            reference_class(Masks(0))(4, 32, 1, 1, 0.5)(X, ei, None)
        assert str(ours.value) == str(ref.value)


@pytest.mark.parametrize("F,dtype,pdtype,ew,needs_grad,p,bn,want", [
    (4, torch.float32, torch.float32, None, False, 0.5, None, True),
    (64, torch.float32, torch.float32, "f32", False, 0.0, None, True),
    (4, torch.float32, torch.float32, None, True, 0.5, None, True),
    (4, torch.float32, torch.float32, None, True, 0.5, "no_fused_training", False),
    (4, torch.float32, torch.float32, None, False, 0.5, "no_fused_training", True),
    (4, torch.float32, torch.float32, None, True, 0.5, "frozen", True),
    (4, torch.float32, torch.float32, None, False, 0.5, "f64_stats", False),
    (4, torch.float32, torch.float32, None, False, 0.5, "strided_stats", False),
    (4, torch.float64, torch.float32, None, False, 0.5, None, False),
    (4, torch.float32, torch.float64, None, False, 0.5, None, False),
    (4, torch.float32, torch.float32, "f64", False, 0.5, None, False),
    (4, torch.float32, torch.float32, "grad", False, 0.5, None, False),
    (4, torch.float32, torch.float32, "2d", False, 0.5, None, False),
    (4, torch.float32, torch.float32, None, False, 1.0, None, False),
    (4, torch.float32, torch.float32, None, False, 0.5, "no_affine", False),
    (4, torch.float32, torch.float32, None, False, 0.5, "no_stats", False),
    (4, torch.float32, torch.float32, None, False, 0.5, "mixed_mode", False),
    (5, torch.float32, torch.float32, None, False, 0.5, None, False)])
def test_routing_predicate(F, dtype, pdtype, ew, needs_grad, p, bn, want):
    m = MPNNLSTM(4 if F == 5 else F, 32, 20, 1, p).to(pdtype)
    if bn == "no_affine":
        m._batch_norm_2 = torch.nn.BatchNorm1d(32, affine=False)
    elif bn == "no_stats":
        m._batch_norm_1 = torch.nn.BatchNorm1d(32, track_running_stats=False)
    elif bn == "mixed_mode":
        m._batch_norm_1.eval()
    elif bn == "no_fused_training":
        m.fused_training = False
    elif bn == "frozen":                     # module in training mode (dropout), both BatchNorms frozen
        m._batch_norm_1.eval()
        m._batch_norm_2.eval()
    elif bn == "f64_stats":
        m._batch_norm_2.running_var = m._batch_norm_2.running_var.double()
    elif bn == "strided_stats":
        m._batch_norm_1.running_mean = torch.zeros(64)[::2]
    X = torch.zeros(20, F, dtype=dtype)
    w = {None: None, "f32": torch.ones(7), "f64": torch.ones(7, dtype=torch.float64), "grad": torch.ones(7, requires_grad=True),
         "2d": torch.ones(7, 1)}[ew]
    assert m._fused_ok(X, w, needs_grad) is want
    assert m._fused_ok(X.unsqueeze(0), None, False) is False
