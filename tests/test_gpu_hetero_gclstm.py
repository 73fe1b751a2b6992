"""HeteroGCLSTM on the GPU: the goldens on the fused route (inference) and op for op (outputs and gradients), the reference's unit test,
bipartite plans against a CPU construction, the fused kernel against float64 across its envelope, determinism, one launch whatever the
number of node types, CUDA-graph replay, routing and the ABI's errors."""
import os

import numpy as np
import pytest
import torch

from hetero_gclstm_seq import CASES, build, fingerprint_close, load, run
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.hetero import HeteroGCLSTM
from pytorch_geometric_temporal_b200.plan import BipartitePlan
from pytorch_geometric_temporal_b200.signal import StaticHeteroGraphTemporalSignal

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda"


def launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


@pytest.mark.parametrize("name", list(CASES))
def test_goldens_fused_inference(name):
    case, gold = CASES[name], load(GOLDEN)[name]
    m, inputs, metadata, _ = build(HeteroGCLSTM, case, DEV, torch.float32)
    with torch.no_grad():
        outs, _, loss = run(m, case, inputs, metadata, DEV, torch.float32, StaticHeteroGraphTemporalSignal, grad=False)
    assert abs(float(loss) - float(gold["loss"])) <= 1e-4 * abs(float(gold["loss"]))
    for k, v in outs.items():
        assert fingerprint_close(v, gold["fingerprints"][k], 1e-4), k


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", list(CASES))
def test_goldens_training(name, fused):
    case, gold = CASES[name], load(GOLDEN)[name]
    m, inputs, metadata, _ = build(HeteroGCLSTM, case, DEV, torch.float32)
    m.fused_training = fused
    outs, grads, loss = run(m, case, inputs, metadata, DEV, torch.float32, StaticHeteroGraphTemporalSignal)
    assert abs(float(loss) - float(gold["loss"])) <= 1e-4 * abs(float(gold["loss"]))
    for k, v in {**outs, **{f"grad.{g}": v for g, v in grads.items()}}.items():
        assert fingerprint_close(v, gold["fingerprints"][k], 1e-4), k


def test_reference_unit_test():
    """The reference's test_hetero_gclstm_layer with its import switched to this package: H None, then carried."""
    g = torch.Generator().manual_seed(0)
    n, feats = 50, {"author": 20, "paper": 30}
    w = (torch.rand(n, n, generator=g) < 0.1).triu(1).nonzero().t().to(DEV)
    ei = {("author", "writes", "paper"): w, ("paper", "rev_writes", "author"): w.flip(0)}
    x = {t: torch.rand(n, c, generator=g).to(DEV) for t, c in feats.items()}
    layer = HeteroGCLSTM(in_channels_dict=feats, out_channels=32, metadata=(list(feats), list(ei))).to(DEV)
    h, c = layer(x, ei)
    assert all(v.shape == (n, 32) for d in (h, c) for v in d.values()) and list(h) == ["author", "paper"]
    h, c = layer(x, ei, h, c)
    assert all(v.shape == (n, 32) for d in (h, c) for v in d.values())


def test_bipartite_plan_matches_cpu_construction():
    g = torch.Generator().manual_seed(3)
    ns, nd = 70, 33
    ei = torch.stack([torch.randint(0, ns, (300,), generator=g), torch.randint(0, nd - 3, (300,), generator=g)])
    ei = torch.cat([ei, ei[:, :20]], 1)
    p = BipartitePlan(ei.to(DEV), ns, nd)
    rowptr, col, val, eid = (t.cpu() for t in p.export(0))
    order = torch.sort(ei[1], stable=True).indices
    cnt = torch.bincount(ei[1], minlength=p.num_nodes)
    assert torch.equal(rowptr, torch.cat([torch.zeros(1, dtype=torch.int64), cnt.cumsum(0)]).int())
    assert torch.equal(eid, order.int()) and torch.equal(col, ei[0][order].int())
    assert torch.equal(val, (1.0 / cnt[ei[1][order]].float()))
    rowptr, col, val, eid = (t.cpu() for t in p.export(0, transposed=True))
    order = torch.sort(ei[0], stable=True).indices
    assert torch.equal(eid, order.int()) and torch.equal(col, ei[1][order].int())
    for bad in ([[ns], [0]], [[0], [nd]], [[-1], [0]]):
        with pytest.raises(RuntimeError):
            BipartitePlan(torch.tensor(bad, device=DEV), ns, nd)


def _graph(types, edges, g):
    """x_dict, edge_index_dict, metadata: types {name: (N, in)}, edges [(src, rel, dst, E)] with in- and out-hubs."""
    x = {t: torch.randn(n, c, generator=g).to(DEV) for t, (n, c) in types.items()}
    ei = {}
    for s, r, d, E in edges:
        ns, nd = types[s][0], types[d][0]
        e = torch.stack([torch.randint(0, ns, (E,), generator=g), torch.randint(0, nd, (E,), generator=g)])
        if E > 8:
            e[1, : E // 8] = 0                                         # an in-hub
            e[0, E // 8: E // 4] = ns - 1                              # an out-hub
        ei[(s, r, d)] = e.to(DEV)
    return x, ei, (list(types), list(ei))


def _oracle(m, x, ei, h, c):
    """The module's op-for-op algebra in float64 on the same parameters."""
    m64 = HeteroGCLSTM(m.in_channels_dict, m.out_channels, m.metadata).to(DEV).double()
    m64.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    d64 = lambda d: None if d is None else {k: v.double() for k, v in d.items()}
    with torch.no_grad():
        return m64(d64(x), ei, d64(h), d64(c))


ENVELOPE = [
    (32, {"a": (1, 1), "b": (2, 32)}, [("a", "r", "b", 3), ("b", "r", "a", 2)]),
    (32, {"a": (33, 31), "b": (31, 7), "c": (4225, 16)}, [("a", "r", "b", 90), ("b", "r", "c", 5000), ("c", "r", "c", 9000),
                                                         ("a", "r", "c", 0), ("c", "r2", "c", 400), ("c", "r", "a", 3000)]),
    (64, {"a": (50000, 9), "b": (32, 1)}, [("b", "r", "a", 60000), ("a", "r", "b", 200)]),
    (32, {f"t{i}": (20 + 13 * i, 1 + 7 * i) for i in range(5)}, [(f"t{i}", "r", f"t{(i + 1) % 5}", 40 + 10 * i) for i in range(5)]
     + [("t0", "s", "t0", 30)]),
]


@pytest.mark.parametrize("case", range(len(ENVELOPE)))
@pytest.mark.parametrize("state", ["none", "h", "hc"])
def test_fused_against_float64(case, state):
    out, types, edges = ENVELOPE[case]
    g = torch.Generator().manual_seed(case)
    x, ei, md = _graph(types, edges, g)
    m = HeteroGCLSTM({t: c for t, (_, c) in types.items()}, out, md).to(DEV)
    h = None if state == "none" else {t: torch.randn(n, out, generator=g).to(DEV) for t, (n, _) in types.items()}
    c = None if state != "hc" else {t: torch.randn(n, out, generator=g).to(DEV) for t, (n, _) in types.items()}
    with torch.no_grad():
        m(x, ei)                                                       # the first call builds the plans and packs the weights
        (hf, cf), nl = launches(lambda: m(x, ei, h, c))
    assert nl == 1
    h64, c64 = _oracle(m, x, ei, h, c)
    for got, want in ((hf, h64), (cf, c64)):
        assert list(got) == list(want)
        for t in want:
            err = (got[t].double() - want[t]).abs().max().item()
            assert err <= 2e-5 * (1 + want[t].abs().max().item()), (t, err)


def test_sequence_repeatable_and_one_launch_per_step():
    out, types, edges = ENVELOPE[3]
    g = torch.Generator().manual_seed(9)
    x, ei, md = _graph(types, edges, g)
    m = HeteroGCLSTM({t: c for t, (_, c) in types.items()}, out, md).to(DEV)
    m(x, ei)                                                           # plans and packs are set up by the first call

    def seq():
        h = c = None
        for _ in range(5):
            h, c = m(x, ei, h, c)
        return h, c
    with torch.no_grad():
        (h1, c1), nl = launches(seq)
        h2, c2 = seq()
    assert nl == 5
    assert all(torch.equal(h1[t], h2[t]) and torch.equal(c1[t], c2[t]) for t in h1)


def test_cuda_graph_replay_of_a_sequence():
    out, types, edges = ENVELOPE[1]
    g = torch.Generator().manual_seed(4)
    x, ei, md = _graph(types, edges, g)
    m = HeteroGCLSTM({t: c for t, (_, c) in types.items()}, out, md).to(DEV)

    def seq():
        h = c = None
        for _ in range(4):
            h, c = m(x, ei, h, c)
        return h
    with torch.no_grad():
        want = seq()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            seq()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            got = seq()
        graph.replay()
        torch.cuda.synchronize()
    assert all(torch.equal(got[t], want[t]) for t in want)


def test_routing():
    g = torch.Generator().manual_seed(5)
    types = {"a": (10, 4), "b": (12, 33)}
    x, ei, md = _graph(types, [("a", "r", "b", 20), ("b", "r", "a", 20)], g)
    m = HeteroGCLSTM({"a": 4, "b": 33}, 32, md).to(DEV)
    with torch.no_grad():
        _, nl = launches(lambda: m(x, ei))
    assert nl > 1                                                      # in_channels 33: op for op
    m = HeteroGCLSTM({"a": 4, "b": 33}, 48, md).to(DEV)
    assert not m._fused_ok(x, None, None, ["a"], {"a": [("b", "r", "a")]}, False)
    m = HeteroGCLSTM({"a": 4, "b": 3}, 64, md).to(DEV)
    inc = {"a": [("b", "r", "a"), ("b", "s", "a")]}
    assert not m._fused_ok({"a": x["a"]}, None, None, ["a"], inc, False)   # out 64 takes one incoming edge type
    assert m._fused_ok({"a": x["a"]}, None, None, ["a"], {"a": inc["a"][:1]}, False)
    assert m._fused_ok({"a": x["a"]}, None, None, ["a"], {"a": inc["a"][:1]}, True)       # training, every type an output
    assert not m._fused_ok(x, None, None, ["a"], {"a": inc["a"][:1]}, True)               # training with "b" not an output
    m.fused_training = False
    assert not m._fused_ok({"a": x["a"]}, None, None, ["a"], {"a": inc["a"][:1]}, True)


def test_abi_errors():
    L = _lib.lib()
    assert L.stmp_hetero_lstm_supported(32, 32, 4) == 1 and L.stmp_hetero_lstm_supported(32, 33, 1) == 0
    assert L.stmp_hetero_lstm_supported(64, 8, 2) == 0 and L.stmp_hetero_lstm_supported(32, 8, 0) == 0
    desc = (torch.zeros(_lib.HETERO_DESC, dtype=torch.int64)).numpy()
    p = desc.ctypes.data_as(__import__("ctypes").c_void_p)
    assert L.stmp_hetero_lstm_fwd(32, 0, p, 0, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_hetero_lstm_fwd(32, 9, p, 0, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_hetero_lstm_fwd(48, 1, p, 0, None) == _lib.STMP_EUNSUPPORTED
    desc[:3] = [4, 3, 1]
    assert L.stmp_hetero_lstm_fwd(32, 1, p, 0, None) == _lib.STMP_EINVAL         # NULL tensors
    assert L.stmp_hetero_lstm_fwd(32, 1, None, 0, None) == _lib.STMP_EINVAL


# ---- training ------------------------------------------------------------------------------------------------------------------------
def _check_err(errs, got, ref32, ref64, what, allow=4):
    """tests/test_gpu_rows_envelope.py's criterion: the fused tensor within `allow` x the fp32 op-for-op error plus 2^-20 of scale."""
    got, ref32, ref64 = got.detach().double(), ref32.detach().double(), ref64.detach()
    e, e32 = float((got - ref64).abs().max()), float((ref32 - ref64).abs().max())
    floor = 2.0 ** -20 * float(ref64.abs().max())
    if not (bool(torch.isfinite(got).all()) and e <= allow * e32 + floor):
        errs.append((what, e, e32, floor))


def _train_call(m, x, ei, h, c, wants, dtype=torch.float32):
    """One call and the gradients of a weighted sum of H' and C' w.r.t. the wanted leaves (x, h, c) and every parameter."""
    cast = lambda d, want: None if d is None else {t: v.to(dtype).detach().requires_grad_(want) for t, v in d.items()}
    xs, hs, cs = cast(x, wants[0]), cast(h, wants[1]), cast(c, wants[2])
    ho, co = m(xs, ei, hs, cs)
    loss = sum((v * (1 + 0.01 * i)).sum() for i, v in enumerate(list(ho.values()) + list(co.values())))
    leaves = {}
    for name, d, want in (("x", xs, wants[0]), ("h", hs, wants[1]), ("c", cs, wants[2])):
        if d is not None and want:
            leaves.update({f"d{name}.{t}": v for t, v in d.items()})
    leaves.update({f"p.{k}": v for k, v in m.named_parameters()})
    g = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    out = {f"h.{t}": v for t, v in ho.items()} | {f"c.{t}": v for t, v in co.items()}
    return out | {k: (torch.zeros_like(v) if gv is None else gv) for (k, v), gv in zip(leaves.items(), g)}


def _clone(m, dtype):
    m2 = HeteroGCLSTM(m.in_channels_dict, m.out_channels, m.metadata).to(DEV, dtype)
    m2.load_state_dict({k: v.to(dtype) for k, v in m.state_dict().items()})
    return m2


TRAIN_CASES = [ENVELOPE[0], ENVELOPE[1], ENVELOPE[2], ENVELOPE[3]]


@pytest.mark.parametrize("case", range(len(TRAIN_CASES)))
@pytest.mark.parametrize("state", ["none", "h", "hc"])
def test_fused_training_against_float64(case, state):
    out, types, edges = TRAIN_CASES[case]
    g = torch.Generator().manual_seed(20 + case)
    x, ei, md = _graph(types, edges, g)
    m = HeteroGCLSTM({t: c for t, (_, c) in types.items()}, out, md).to(DEV)
    m(x, ei)
    h = None if state == "none" else {t: torch.randn(n, out, generator=g).to(DEV) for t, (n, _) in types.items()}
    c = None if state != "hc" else {t: torch.randn(n, out, generator=g).to(DEV) for t, (n, _) in types.items()}
    subsets = [(a, b, d) for a in (False, True) for b in (False, True) for d in (False, True)] if case == 1 else [(True, True, True)]
    for wants in subsets:
        got, nl = launches(lambda: _train_call(m, x, ei, h, c, wants))
        assert nl <= 1 + 4, nl
        op = _clone(m, torch.float32)
        op.fused_training = False
        ref32 = _train_call(op, x, ei, h, c, wants)
        ref64 = _train_call(_clone(m, torch.float64), x, ei, h, c, wants, torch.float64)
        errs = []
        for k in ref64:
            _check_err(errs, got[k], ref32[k], ref64[k], (wants, k))
        assert not errs, errs[:5]
        if h is None:                                                  # no state: the lin_l / lin_r weights get exact zeros
            assert all(float(v.abs().max()) == 0 for k, v in got.items() if ".lin_" in k and k.endswith("weight"))


def test_cin_sweep_against_float64():
    """Every in_channels 1..32, on both sides of each 32-column group of the basis (nb = in + 32 (1 + R), R = 1..3)."""
    errs = []
    for cin in range(1, 33):
        R = 1 + cin % 3
        g = torch.Generator().manual_seed(100 + cin)
        edges = [("a", "r", "b", 200)] + [("b", f"s{k}", "b", 100 + k) for k in range(R - 1)] + [("b", "r", "a", 150)]
        x, ei, md = _graph({"a": (33, cin), "b": (31, 33 - cin)}, edges, g)
        m = HeteroGCLSTM({"a": cin, "b": 33 - cin}, 32, md).to(DEV)
        h = {t: torch.randn(v.size(0), 32, generator=g).to(DEV) for t, v in x.items()}
        got = _train_call(m, x, ei, h, h, (True, True, True))
        op = _clone(m, torch.float32)
        op.fused_training = False
        ref32, ref64 = _train_call(op, x, ei, h, h, (True, True, True)), _train_call(_clone(m, torch.float64), x, ei, h, h, (True,) * 3,
                                                                                      torch.float64)
        for k in ref64:
            _check_err(errs, got[k], ref32[k], ref64[k], (cin, k))
    assert not errs, errs[:5]


@pytest.mark.parametrize("ntypes", [2, 5])
def test_training_bit_equal_repeatable_equivariant_and_launches(ntypes):
    out, types, edges = ENVELOPE[0] if ntypes == 2 else ENVELOPE[3]
    g = torch.Generator().manual_seed(7)
    x, ei, md = _graph(types, edges, g)
    m = HeteroGCLSTM({t: c for t, (_, c) in types.items()}, out, md).to(DEV)
    h = {t: torch.randn(n, out, generator=g).to(DEV) for t, (n, _) in types.items()}
    m(x, ei)
    with torch.no_grad():
        h_ng, c_ng = m(x, ei, h, h)
    xs = {t: v.clone().requires_grad_() for t, v in x.items()}
    hs = {t: v.clone().requires_grad_() for t, v in h.items()}
    (ho, co), nf = launches(lambda: m(xs, ei, hs, hs))
    assert nf == 1
    assert all(torch.equal(ho[t], h_ng[t]) and torch.equal(co[t], c_ng[t]) for t in ho)
    loss = sum(v.square().sum() for v in list(ho.values()) + list(co.values()))
    leaves = list(xs.values()) + list(hs.values()) + list(m.parameters())
    g1, nb = launches(lambda: torch.autograd.grad(loss, leaves, retain_graph=True))
    assert nb == 4
    g2 = torch.autograd.grad(loss, leaves, retain_graph=True)
    g3 = torch.autograd.grad(2 * loss, leaves)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    assert all(torch.equal(2 * a, b) for a, b in zip(g1, g3))


@pytest.mark.parametrize("fused", [True, False])
def test_cuda_graph_training_step(fused):
    out, types, edges = ENVELOPE[1]
    g = torch.Generator().manual_seed(8)
    x, ei, md = _graph(types, edges, g)
    m = HeteroGCLSTM({t: c for t, (_, c) in types.items()}, out, md).to(DEV)
    m.fused_training = fused
    with torch.no_grad():
        m(x, ei)                                                       # plans and packs, with no autograd graph left behind
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)

    def grads():
        opt.zero_grad(set_to_none=False)
        h = c = None
        loss = 0
        for _ in range(3):
            h, c = m(x, ei, h, c)
            loss = loss + sum(v.square().mean() for v in h.values())
        loss.backward()

    def step():
        grads()
        opt.step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    graph.replay()                                                     # gradients at `state`, then the Adam step
    torch.cuda.synchronize()
    replayed = {k: p.grad.clone() for k, p in m.named_parameters()}
    assert any(not torch.equal(v, state[k]) for k, v in m.state_dict().items())
    m.load_state_dict(state)
    grads()                                                            # the same gradients, eager
    torch.cuda.synchronize()
    for k, p in m.named_parameters():
        assert torch.equal(p.grad, replayed[k]) if fused else torch.allclose(p.grad, replayed[k], rtol=1e-5, atol=1e-7), k
