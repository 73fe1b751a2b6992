"""HeteroGCLSTM host-side checks: the restated PyG layers driving the unmodified reference against the goldens, state_dict layout and
seeded lazy materialisation against the reference, loading a reference state_dict, the reference's errors, and
StaticHeteroGraphTemporalSignal / HeteroData (the reference's signal tests, restated)."""
import os

import numpy as np
import pytest
import torch

from hetero_gclstm_seq import CASES, build, fingerprint_close, load, materialize_reference, reference_class, run
from oracle import refload
from pytorch_geometric_temporal_b200.nn.hetero import HeteroGCLSTM
from pytorch_geometric_temporal_b200.signal import HeteroData, StaticHeteroGraphTemporalSignal, temporal_signal_split

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
needs_ref = pytest.mark.skipif(not refload.available(), reason="reference tree not present")


@pytest.fixture
def f64():
    d = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(d)


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_reference_on_restated_layers_matches_goldens(name, f64):
    case, gold = CASES[name], load(GOLDEN)[name]
    m, inputs, metadata, _ = build(reference_class(), case)
    materialize_reference(m, inputs, metadata)
    outs, grads, loss = run(m, case, inputs, metadata, "cpu", torch.float64, StaticHeteroGraphTemporalSignal)
    assert torch.equal(loss, gold["loss"])
    got = {**outs, **{f"grad.{k}": v for k, v in grads.items()}}
    assert set(got) == set(gold["fingerprints"])
    for k, v in got.items():
        assert fingerprint_close(v, gold["fingerprints"][k], 1e-12), k


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_state_dict_and_seeded_materialisation_match_reference(name, f64):
    case = CASES[name]
    _, inputs, metadata, cin = build(reference_class(), case)
    fresh_ref, fresh = reference_class()(cin, case["out"], metadata), HeteroGCLSTM(cin, case["out"], metadata)
    assert list(fresh.state_dict()) == list(fresh_ref.state_dict())    # keys and order before materialisation
    materialize_reference(ref := build(reference_class(), case)[0], inputs, metadata)   # right after its seeded construction
    ours = build(HeteroGCLSTM, case)[0]                                 # construction + HeteroGCLSTM.materialize on the CPU
    sd_ref, sd = ref.state_dict(), ours.state_dict()
    assert list(sd) == list(sd_ref)
    for k in sd_ref:
        assert torch.equal(sd[k], sd_ref[k]), k


@needs_ref
def test_loading_a_reference_state_dict(f64):
    case = CASES["three32"]
    ref, inputs, metadata, cin = build(reference_class(), case)
    materialize_reference(ref, inputs, metadata)
    m = HeteroGCLSTM(cin, case["out"], metadata)
    m.load_state_dict(ref.state_dict())
    for k, v in ref.state_dict().items():
        assert torch.equal(m.state_dict()[k], v)
    assert m.conv_o.conv(("a", "to", "b")).lin_l.in_channels == case["out"]


def test_state_dict_keys():
    m = HeteroGCLSTM({"a": 3, "b": 4}, 32, (["a", "b"], [("a", "to", "b"), ("b", "rev", "a")]), bias=False)
    keys = list(m.state_dict())
    assert keys[:5] == ["conv_i.convs.<a___to___b>.lin_l.weight", "conv_i.convs.<a___to___b>.lin_r.weight",
                        "conv_i.convs.<b___rev___a>.lin_l.weight", "conv_i.convs.<b___rev___a>.lin_r.weight", "W_i.a"]
    assert keys[5:7] == ["W_i.b", "b_i.a"] and m.b_i["a"].shape == (1, 32)


def _small():
    m = HeteroGCLSTM({"a": 3, "b": 4}, 32, (["a", "b"], [("a", "to", "b"), ("b", "rev", "a"), ("b", "x", "b")]))
    x = {"a": torch.randn(5, 3), "b": torch.randn(6, 4)}
    ei = {("a", "to", "b"): torch.tensor([[0, 1], [2, 3]]), ("b", "rev", "a"): torch.tensor([[0], [1]])}
    return m, x, ei


def test_errors_before_any_launch():
    m, x, ei = _small()
    with pytest.raises(KeyError):                      # a type without a W_* entry
        m({**x, "z": torch.randn(2, 1)}, ei)
    with pytest.raises(KeyError):                      # "a" has no incoming edge type once ("b", "rev", "a") is absent
        m(x, {("a", "to", "b"): ei[("a", "to", "b")]})
    with pytest.raises(RuntimeError, match="channels"):
        m({"a": torch.randn(5, 2), "b": x["b"]}, ei)
    with pytest.raises(RuntimeError, match="h_dict"):
        m(x, ei, {"a": torch.randn(5, 31), "b": torch.randn(6, 32)})
    with pytest.raises(RuntimeError, match="CUDA only"):   # CPU tensors are refused, after every shape check
        m(x, ei)
    # edge types of edge_index_dict outside the metadata are ignored, and ones of the metadata missing from it are skipped
    assert m._edges({**ei, ("a", "new", "a"): ei[("b", "rev", "a")]}) == [("a", "to", "b"), ("b", "rev", "a")]


def test_signal_snapshots_and_split():
    ei = {("author", "writes", "paper"): np.array([[0, 0, 1], [0, 1, 2]])}
    feats = [{"author": np.full((2, 1), t / 10), "paper": np.full((3, 1), t / 10)} for t in range(3)]
    targets = [{"author": np.array([t, t]), "paper": np.array([t, t, t])} for t in range(3)]
    extra = [{"author": np.ones((2, 2)), "paper": None} for _ in range(3)]
    sig = StaticHeteroGraphTemporalSignal(ei, None, feats, targets, extra=extra)
    assert sig.snapshot_count == 3
    snaps = list(sig)
    assert len(snaps) == 3 and all(isinstance(s, HeteroData) for s in snaps)
    s = snaps[1]
    assert s.node_types == ["author", "paper"] and s.edge_types == [("author", "writes", "paper")]
    assert s["author"].x.dtype == torch.float32 and s["paper"].y.dtype == torch.int64
    assert torch.equal(s["author"].extra, torch.ones(2, 2)) and "extra" not in s["paper"]
    assert s.metadata() == (["author", "paper"], [("author", "writes", "paper")])
    assert snaps[0].edge_index_dict[("author", "writes", "paper")] is snaps[2].edge_index_dict[("author", "writes", "paper")]
    train, test = temporal_signal_split(sig, train_ratio=0.67)
    assert train.snapshot_count == 2 and test.snapshot_count == 1
    assert torch.equal(test[0]["paper"].x, torch.full((3, 1), 0.2, dtype=torch.float32))
    skipped = StaticHeteroGraphTemporalSignal(ei, None, [feats[0], None, {"author": feats[2]["author"], "paper": None}], targets)
    assert skipped[1].x_dict == {} and list(skipped[2].x_dict) == ["author"]


def test_backward_decomposition_against_autograd():
    """The fused backward's algebra in float64: dpre from the gates, dS = dpre w on the packed basis, dX and the own-row dH from its
    blocks, Q_e = its mean blocks, dH_s += Op_e^T Q_e, dw = dpre^T S and db = sum dpre, with the summed roots handed to every lin_r^e and
    the summed bias to b_g and every lin_l^e.bias."""
    torch.manual_seed(0)
    D, out = torch.float64, 8
    n = {"a": 7, "b": 5}
    cin = {"a": 3, "b": 4}
    ei = {("a", "r", "b"): torch.tensor([[0, 1, 6, 6, 2], [0, 0, 4, 4, 1]]), ("b", "s", "b"): torch.tensor([[0, 4, 3], [1, 1, 2]]),
          ("b", "r", "a"): torch.tensor([[1, 2, 2], [6, 0, 0]])}
    inc = {"a": [("b", "r", "a")], "b": [("a", "r", "b"), ("b", "s", "b")]}
    op = lambda e: torch.zeros(n[e[2]], n[e[0]], dtype=D).index_put_((ei[e][1], ei[e][0]), torch.ones(ei[e].size(1), dtype=D),
                                                                     accumulate=True)
    Op = {e: (lambda A: A / A.sum(1, keepdim=True).clamp(min=1))(op(e)) for e in ei}
    x = {t: torch.randn(n[t], cin[t], dtype=D, requires_grad=True) for t in n}
    h = {t: torch.randn(n[t], out, dtype=D, requires_grad=True) for t in n}
    c = {t: torch.randn(n[t], out, dtype=D, requires_grad=True) for t in n}
    W = {t: torch.randn(4, cin[t], out, dtype=D, requires_grad=True) for t in n}
    bb = {t: torch.randn(4, out, dtype=D, requires_grad=True) for t in n}
    ll = {e: torch.randn(4, out, out, dtype=D, requires_grad=True) for e in ei}
    lb = {e: torch.randn(4, out, dtype=D, requires_grad=True) for e in ei}
    lr = {e: torch.randn(4, out, out, dtype=D, requires_grad=True) for e in ei}
    gh = {t: torch.randn(n[t], out, dtype=D) for t in n}
    gc = {t: torch.randn(n[t], out, dtype=D) for t in n}
    fwd = {}
    for t in n:
        pre = [x[t] @ W[t][g] + bb[t][g] + sum(Op[e] @ h[e[0]] @ ll[e][g].t() + lb[e][g] + h[t] @ lr[e][g].t() for e in inc[t])
               for g in range(4)]
        I, F, T, O = torch.sigmoid(pre[0]), torch.sigmoid(pre[1]), torch.tanh(pre[2]), torch.sigmoid(pre[3])
        cn = F * c[t] + I * T
        fwd[t] = (I, F, T, O, cn, O * torch.tanh(cn))
    loss = sum((fwd[t][5] * gh[t]).sum() + (fwd[t][4] * gc[t]).sum() for t in n)
    leaves = [*x.values(), *h.values(), *c.values(), *W.values(), *bb.values(), *ll.values(), *lb.values(), *lr.values()]
    auto = dict(zip(range(len(leaves)), torch.autograd.grad(loss, leaves)))
    auto = iter(auto.values())
    ax, ah, ac = ({t: next(auto) for t in n} for _ in range(3))
    aW, ab = ({t: next(auto) for t in n} for _ in range(2))
    all_, alb, alr = ({e: next(auto) for e in ei} for _ in range(3))
    dh = {}
    Q = {}
    with torch.no_grad():
        for t in n:
            I, F, T, O, cn, _ = fwd[t]
            tc = torch.tanh(cn)
            dcn = gc[t] + gh[t] * O * (1 - tc * tc)
            dpre = torch.cat([dcn * T * I * (1 - I), dcn * c[t] * F * (1 - F), dcn * I * (1 - T * T), gh[t] * tc * O * (1 - O)], 1)
            w = torch.cat([torch.cat([W[t][g].t(), sum(lr[e][g] for e in inc[t])] + [ll[e][g] for e in inc[t]], 1) for g in range(4)])
            S = torch.cat([x[t], h[t]] + [Op[e] @ h[e[0]] for e in inc[t]], 1)
            dS = dpre @ w
            assert torch.allclose(dS[:, :cin[t]], ax[t])
            assert torch.allclose(dcn * F, ac[t])
            dh[t] = dS[:, cin[t]:cin[t] + out].clone()
            for r, e in enumerate(inc[t]):
                Q[e] = dS[:, cin[t] + out * (1 + r):cin[t] + out * (2 + r)]
            dw, db = dpre.t() @ S, dpre.sum(0)
            for g in range(4):
                rows = slice(g * out, (g + 1) * out)
                assert torch.allclose(dw[rows, :cin[t]].t(), aW[t][g]) and torch.allclose(db[rows], ab[t][g])
                for r, e in enumerate(inc[t]):
                    assert torch.allclose(dw[rows, cin[t]:cin[t] + out], alr[e][g])          # the summed root's block, to every lin_r^e
                    assert torch.allclose(dw[rows, cin[t] + out * (1 + r):cin[t] + out * (2 + r)], all_[e][g])
                    assert torch.allclose(db[rows], alb[e][g])                              # the summed bias's gradient, to every lin_l^e.bias
        for e in ei:                                                                        # the transposed means, in metadata order
            dh[e[0]] = dh[e[0]] + Op[e].t() @ Q[e]
        for t in n:
            assert torch.allclose(dh[t], ah[t])
