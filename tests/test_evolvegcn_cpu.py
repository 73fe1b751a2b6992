"""EvolveGCNO / EvolveGCNH without a GPU: the float64 oracle against the reference's stored results, the state_dict keys and seeded
initialisation against the reference's, TopKPooling's k and the k != C error against the reference, the routing predicate and the mapping
from constructor flags to plans."""
import os

import pytest
import torch

from evolvegcn_seq import TopKPooling, check_reference, graph_of, load, oracle_run, reference_classes, topk_k
from oracle import refload
from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.nn.recurrent import EvolveGCNH, EvolveGCNO
from pytorch_geometric_temporal_b200.nn.recurrent.evolvegcn import topk_size

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
D = torch.float64


@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_oracle_matches_reference(name):
    c = load(GOLDEN)["cases"][name]
    ei, ew, X, Y = graph_of(c, GOLDEN)
    outs, cost, leaves = oracle_run(c, X, Y, ei, ew, c["epochs"])
    check_reference(c, outs.detach(), cost, {k: v.grad for k, v in leaves.items()})


KEYS_O = ["initial_weight"] + [f"recurrent_layer.{p}_l0" for p in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


@pytest.mark.parametrize("kind,C,nodes", [("O", 4, None), ("O", 32, None), ("H", 4, 20), ("H", 14, 1068), ("H", 33, 40)])
def test_state_dict_and_seeded_init_match_reference(kind, C, nodes):
    ours = EvolveGCNH(nodes, C) if kind == "H" else EvolveGCNO(C)
    want = KEYS_O[:1] + (["pooling_layer.select.weight"] if kind == "H" else []) + KEYS_O[1:]
    assert list(ours.state_dict()) == want
    assert isinstance(ours.recurrent_layer, torch.nn.GRU) and ours.weight is None
    if not refload.available():
        pytest.skip("reference tree not present")
    ref_o, ref_h = reference_classes()
    for flags in ({}, dict(improved=True, normalize=False, add_self_loops=False)):
        torch.manual_seed(11)
        ref = ref_h(nodes, C, **flags) if kind == "H" else ref_o(C, **flags)
        torch.manual_seed(11)
        ours = EvolveGCNH(nodes, C, **flags) if kind == "H" else EvolveGCNO(C, **flags)
        assert list(ref.state_dict()) == list(ours.state_dict())
        for k, v in ref.state_dict().items():
            assert torch.equal(v, ours.state_dict()[k]), k


def test_draw_order():
    """TopKPooling's weight (drawn twice), then the GRU, then glorot(initial_weight)."""
    torch.manual_seed(5)
    m = EvolveGCNH(20, 4)
    torch.manual_seed(5)
    torch.empty(1, 4).uniform_(-0.5, 0.5)
    p = torch.empty(1, 4).uniform_(-0.5, 0.5)
    gru = torch.nn.GRU(4, 4)
    a = (6.0 / 8) ** 0.5
    w = torch.empty(1, 4, 4).uniform_(-a, a)
    assert torch.equal(m.pooling_layer.select.weight, p) and torch.equal(m.initial_weight, w)
    for k, v in gru.state_dict().items():
        assert torch.equal(getattr(m.recurrent_layer, k), v), k


@pytest.mark.parametrize("N,C,dtype", [(21, 3, torch.float32), (39, 5, torch.float32), (1033, 17, torch.float32), (20, 20, torch.float32),
                                       (20, 4, torch.float32), (1068, 14, torch.float32), (21, 3, torch.float64), (7, 2, torch.float32),
                                       (3, 5, torch.float32), (100, 8, torch.float64)])
def test_k_and_the_k_error_against_reference(N, C, dtype):
    """k = ceil(ratio N) in X's dtype (int(ratio) when ratio >= 1, (20, 20)), at most N; the module raises RuntimeError before any launch
    where k != C, as the reference's GRU does.  (7, 2): the module built for 2 of 7 nodes; (3, 5): fewer nodes than C."""
    ratio = C / N
    assert topk_size(ratio, N, dtype) == topk_k(ratio, N, dtype)
    k = topk_size(ratio, N, dtype)
    pool = TopKPooling(C, ratio)
    X = torch.randn(N, C, dtype=dtype)
    assert pool(X, None)[0].size(0) == k
    m = EvolveGCNH(N, C).to(dtype)
    ei = torch.zeros(2, 0, dtype=torch.int64)
    if k != C:
        with pytest.raises(RuntimeError, match="TopKPooling keeps"):
            m(X, ei)
    if refload.available():
        torch.manual_seed(0)
        ref = reference_classes()[1](N, C).to(dtype)
        if k != C:
            with pytest.raises(RuntimeError):
                ref(X, ei)
        else:
            assert ref(X, ei).shape == (N, C)


@pytest.mark.parametrize("ratio,N,want", [(2.0, 10, 2), (1.0, 10, 1), (3.7, 10, 3), (25.0, 10, 10), (0.5, 9, 5)])
def test_k_at_and_above_ratio_one(ratio, N, want):
    assert topk_size(ratio, N, torch.float32) == want == topk_k(ratio, N, torch.float32)


class _Plan:
    num_nodes = 20


@pytest.mark.parametrize("F,C,dtype,wdtype,ew,training,fused,want", [
    (4, 4, torch.float32, torch.float32, None, False, True, True), (32, 32, torch.float32, torch.float32, "f32", True, True, True),
    (33, 33, torch.float32, torch.float32, None, False, True, False), (4, 4, torch.float64, torch.float32, None, False, True, False),
    (4, 4, torch.float32, torch.float64, None, False, True, False), (4, 4, torch.float32, torch.float32, "f64", False, True, False),
    (4, 4, torch.float32, torch.float32, "grad", True, True, False), (4, 4, torch.float32, torch.float32, None, True, False, False),
    (4, 4, torch.float32, torch.float32, None, False, False, True), (5, 4, torch.float32, torch.float32, None, False, True, False)])
def test_routing_predicate(F, C, dtype, wdtype, ew, training, fused, want):
    for m in (EvolveGCNO(C), EvolveGCNH(20, C)):
        m.fused_training = fused
        X = torch.zeros(20, F, dtype=dtype)
        w = {None: None, "f32": torch.ones(7), "f64": torch.ones(7, dtype=torch.float64), "grad": torch.ones(7, requires_grad=True)}[ew]
        assert m._fused_ok(X, m.initial_weight.to(wdtype), w, training) is want
        assert m._fused_ok(X.unsqueeze(0), m.initial_weight, None, training) is False


@pytest.mark.parametrize("normalize,improved,loops,want", [
    (True, False, True, (_lib.FLAVOR_GCN, 0)), (True, True, True, (_lib.FLAVOR_GCN, _lib.GCN_IMPROVED)),
    (True, False, False, (_lib.FLAVOR_GCN, _lib.GCN_NO_SELF_LOOPS)),
    (True, True, False, (_lib.FLAVOR_GCN, _lib.GCN_IMPROVED | _lib.GCN_NO_SELF_LOOPS)), (False, True, False, "gated")])
def test_flags_to_plans(monkeypatch, normalize, improved, loops, want):
    """normalize=True: the GCN plan with improved / add_self_loops as its flags; normalize=False: the add GatedGraphConv plan (the raw
    edge weights), whatever the other two flags say."""
    m = EvolveGCNO(4, improved=improved, normalize=normalize, add_self_loops=loops)
    asked = []
    monkeypatch.setattr(m._plans, "get", lambda flavor, ei, ew, n, flags=0, **kw: asked.append((flavor, flags)) or "plan")
    monkeypatch.setattr(m._plans, "get_gated", lambda ei, ew, n, aggr: asked.append(("gated", aggr)) or "plan")
    assert m._plan(None, None, 20) == "plan"
    assert asked == ([("gated", "add")] if want == "gated" else [want])


def test_weight_attribute_semantics():
    """weight starts None; reinitialize_weight() resets it; it is a plain attribute, not a parameter or buffer."""
    m = EvolveGCNO(4)
    assert m.weight is None and "weight" not in m.state_dict()
    m.weight = torch.zeros(1, 4, 4)
    m.reinitialize_weight()
    assert m.weight is None
