"""DyGrEncoder on the H100: the gated plan bit-exact against a CPU restatement, every golden case fused and op for op against the float64
oracle (held to the reference's fingerprints by tests/test_dygrae_cpu.py), a float64 envelope over aggregations, widths, layers, weights,
states and graph geometries, bit-equal training and inference forwards, repeatable and loss-scale-equivariant gradients, exact launch
counts, the routes outside the envelope, CUDA-graph replay and the ABI's errors."""
import ctypes
import os

import pytest
import torch

from dygrae_seq import dygrae_step, load, model_for, oracle_run, run, states_for
from gconvgru_seq import chickenpox_train_split
from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.nn.recurrent import DyGrEncoder
from pytorch_geometric_temporal_b200.plan import GatedPlan, GraphPlan
from wikimaths_seq import load as load_wikimaths

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
AGGRS = ("add", "mean", "max")


@pytest.fixture(autouse=True)
def _cudnn_fp32():
    """cuDNN's LSTM (the C > 16 and two-layer routes) and the op-for-op path in full fp32: by default torch lets cuDNN round operands to
    TF32, about 1e-3 off the float64 oracle."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _plan_cpu(ei, ew, n, aggr):
    """(rowptr, col, val, eid) by destination and by source: every edge in edge order, val = w (add, max) or w / cnt(dst) (mean)."""
    src, dst = ei[0], ei[1]
    w = torch.ones(ei.size(1)) if ew is None else ew.float()
    if aggr == "mean":
        w = w / torch.bincount(dst, minlength=n).float()[dst]
    out = []
    for key, other in ((dst, src), (src, dst)):
        order = torch.sort(key, stable=True).indices
        rowptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(torch.bincount(key, minlength=n), 0)])
        out.append((rowptr.int(), other[order].int(), w[order].float(), order.int()))
    return out


def _graph_of(kind, n, seed):
    """edge_index of a named geometry on n nodes."""
    g = torch.Generator().manual_seed(seed)
    if kind == "empty":
        return torch.zeros(2, 0, dtype=torch.int64)
    if kind == "one_node":
        return torch.tensor([[0, 0], [0, 0]])                                   # a duplicated self loop on the only node
    e = 4 * n
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, max(1, n - 3), (e,), generator=g)                    # the last nodes have no in-edge
    if kind == "hub":
        dst[:400] = 0                                                           # a 400-edge hub
        src[400:800] = 1                                                        # and a 400-edge source
    ei = torch.stack([src, dst])
    return torch.cat([ei, ei[:, :e // 8], torch.stack([src[:5], src[:5]])], 1)  # duplicates (exact max ties) and self loops


def _weights(kind, E, seed):
    if kind is None:
        return None
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(E, generator=g) * 2
    if kind == "signed":
        w = w - 1
        w[::7] = 0.0                                                            # zero and negative weights
    return w


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("n,kind,wk", [(20, "random", None), (300, "hub", "signed"), (7, "empty", None), (1, "one_node", "pos")])
def test_plan_bit_exact(aggr, n, kind, wk):
    ei = _graph_of(kind, n, n)
    ew = _weights(wk, ei.size(1), 3)
    plan = GatedPlan(ei.to(DEV), None if ew is None else ew.to(DEV), n, aggr)
    assert plan.n_ops == 1
    want = _plan_cpu(ei, ew, n, aggr)
    for t in (0, 1):
        got = [x.cpu() for x in plan.export(0, bool(t))]
        for a, b in zip(got, want[t]):
            assert torch.equal(a, b)


def test_plan_rejects_bad_graphs():
    ei = torch.tensor([[0, 5], [1, 0]], device=DEV)
    with pytest.raises(RuntimeError, match="outside"):
        GatedPlan(ei, None, 3, "add")
    out = ctypes.c_void_p()
    L = _lib.lib()
    assert L.stmp_plan_create_gated(3, 1, _lib.ptr(ei), None, 3, None, ctypes.byref(out)) == _lib.STMP_EINVAL
    assert L.stmp_plan_create(_lib.FLAVOR_GATED, 3, 1, _lib.ptr(ei), None, 0, -1.0, 0, None, ctypes.byref(out)) == _lib.STMP_EINVAL


def _graph(c):
    if c["graph"] == "chickenpox":
        return chickenpox_train_split()
    w = load_wikimaths(GOLDEN)
    return w["edge_index"], w["edge_weight"], w["X"], w["Y"]


def _close(got, want, what, rtol=2e-4):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = float(want.abs().max()) + 1e-30
    err = float((got - want).abs().max()) / scale
    assert err <= rtol, (what, err)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_golden_cases(name, fused):
    c = load(GOLDEN)["cases"][name]
    ei, ew, X, Y = _graph(c)
    H0, C0 = states_for(c, X.shape[1], dtype=torch.float64)
    outs64, cost64, leaves = oracle_run(c, X, Y, ei, ew, H0, C0)
    cost64.backward()
    m = model_for(c, DEV, fused)
    h0, c0 = states_for(c, X.shape[1], DEV)
    before = dict(_lib.path_counters())
    outs, cost = run(m, X.to(DEV), Y.to(DEV), ei.to(DEV), ew.to(DEV), h0, c0, c["state"] != "none")
    cost.backward()
    after = _lib.path_counters()
    ran = lambda k: after.get(k, 0) > before.get(k, 0)
    assert (ran("k_ggc_rows_fwd") or ran("k_ggc_rows_fwd_max")) is fused
    assert (ran("k_lstm_rows_fwd") or ran("k_lstm_wide_rows_fwd")) is (fused and c["C"] <= 16 and c["Ll"] == 1)
    assert abs(float(cost.detach()) - float(cost64.detach())) <= 1e-5 * abs(float(cost64.detach()))
    _close(outs, outs64, "out")
    for k, p in m.named_parameters():
        _close(p.grad, leaves[k].grad, k, 1e-3)
    if H0 is not None:
        _close(h0.grad, H0.grad, "gH0", 1e-3)
        _close(c0.grad, C0.grad, "gC0", 1e-3)


def _params64(m):
    return {k: v.detach().double().cpu().requires_grad_(True) for k, v in m.state_dict().items()}


def _check_step(m, c, X, ei, ew, H, C, want_dx, rtol=1e-3):
    """One fused step (conv route asserted) against dygrae_step in float64: outputs, every parameter's, X's, H's and C's gradient."""
    p64 = _params64(m)
    xs = [None if t is None else t.double().requires_grad_(want_dx or i > 0) for i, t in enumerate((X, H, C))]
    o64 = dygrae_step(p64, c, xs[0], ei, ew, xs[1], xs[2])
    g = torch.Generator().manual_seed(1)
    coef = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in o64]
    sum((a * b).sum() for a, b in zip(o64, coef)).backward()
    md = m.to(DEV)
    xd = [None if t is None else t.to(DEV).requires_grad_(want_dx or i > 0) for i, t in enumerate((X, H, C))]
    before = dict(_lib.path_counters())
    o = md(xd[0], ei.to(DEV), None if ew is None else ew.to(DEV), xd[1], xd[2])
    after = _lib.path_counters()
    assert sum(after.get(k, 0) - before.get(k, 0) for k in ("k_ggc_rows_fwd", "k_ggc_rows_fwd_max")) == c["Lg"]
    sum((a * b.float().to(DEV)).sum() for a, b in zip(o, coef)).backward()
    for a, b, what in zip(o, o64, ("H_tilde", "H", "C")):
        _close(a, b, what, 1e-4)
    for k, q in md.named_parameters():
        _close(q.grad, p64[k].grad, k, rtol)
    for t, ref, what in zip(xd, xs, ("dX", "dH", "dC")):
        if t is not None and t.requires_grad:
            _close(t.grad, ref.grad, what, rtol)


def _model(C, Lg, aggr, Ho, seed):
    torch.manual_seed(seed)
    m = DyGrEncoder(C, Lg, aggr, Ho, 1)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.4)
    return m


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("C", [1, 4, 5, 16, 17, 32])
@pytest.mark.parametrize("Fk", ["one", "full"])
@pytest.mark.parametrize("Lg", [1, 2, 3])
def test_envelope_against_float64(aggr, C, Fk, Lg):
    F = 1 if Fk == "one" else C
    seed = 100 * C + 10 * Lg + F + AGGRS.index(aggr)
    Ho = (32, 64)[seed % 2]
    wk = (None, "pos", "signed")[seed % 3]
    with_state = (seed // 3) % 2 == 0
    n = 37
    ei = _graph_of("random", n, seed)
    ew = _weights(wk, ei.size(1), seed)
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(n, F, generator=g)
    H = torch.randn(n, Ho, generator=g) * 0.5 if with_state else None
    Cs = torch.randn(n, Ho, generator=g) * 0.5 if with_state else None
    c = dict(C=C, Lg=Lg, aggr=aggr, Ho=Ho, Ll=1)
    _check_step(_model(C, Lg, aggr, Ho, seed), c, X, ei, ew, H, Cs, want_dx=seed % 4 != 0)


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("kind,n", [("empty", 9), ("one_node", 1), ("hub", 1200), ("random", 50000)])
def test_graph_geometries(aggr, kind, n):
    """0 edges, one node, isolated nodes, a 400-edge hub and source, duplicate edges (exact max ties: the gradient is split evenly), self
    loops, and 50 000 nodes.  At 50 000 nodes max takes a looser tolerance: two messages within float32 rounding of each other can swap
    the argmax against float64, which moves one message's gradient to the other."""
    ei = _graph_of(kind, n, 7)
    ew = _weights("signed" if kind == "hub" else None, ei.size(1), 7)
    g = torch.Generator().manual_seed(n)
    C, Ho = 16, 32
    X = torch.randn(n, 14, generator=g)
    H, Cs = torch.randn(n, Ho, generator=g) * 0.5, torch.randn(n, Ho, generator=g) * 0.5
    c = dict(C=C, Lg=2, aggr=aggr, Ho=Ho, Ll=1)
    rtol = 2e-2 if (aggr == "max" and n >= 50000) else 1e-3
    _check_step(_model(C, 2, aggr, Ho, n), c, X, ei, ew, H, Cs, want_dx=True, rtol=rtol)


@pytest.mark.parametrize("aggr", AGGRS)
def test_exact_ties_split_the_gradient(aggr):
    """Every edge appears three times: each max is an exact three-way tie in float32 and float64 alike."""
    ei = _graph_of("random", 50, 3)
    ei = torch.cat([ei, ei, ei], 1)
    g = torch.Generator().manual_seed(4)
    X = torch.randn(50, 8, generator=g)
    c = dict(C=8, Lg=2, aggr=aggr, Ho=32, Ll=1)
    _check_step(_model(8, 2, aggr, 32, 5), c, X, ei, None, None, None, want_dx=True)


def _launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("Lg", [1, 3])
def test_training_equals_inference_repeats_and_counts(aggr, Lg):
    """Inference and the training forward: L_g GatedGraphConv launches (one more for max) + one LSTM launch.  Backward: the LSTM cell's
    one + two weight-gradient launches, then L_g GatedGraphConv launches, one more for dX (add, mean) or always (max), and two for its
    weight gradients."""
    m = _model(16, Lg, aggr, 32, 3).to(DEV)
    ei = _graph_of("hub", 700, 3).to(DEV)
    ew = _weights("pos", ei.size(1), 3).to(DEV)
    g = torch.Generator().manual_seed(2)
    X, H, C = torch.randn(700, 14, generator=g).to(DEV), torch.randn(700, 32, generator=g).to(DEV), torch.randn(700, 32, generator=g).to(DEV)
    mx = aggr == "max"
    with torch.no_grad():
        want = m(X, ei, ew, H, C)
        got, n = _launches(lambda: m(X, ei, ew, H, C))
    assert n == Lg + mx + 1
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    out, n = _launches(lambda: m(X, ei, ew, H, C))
    assert n == Lg + mx + 1
    assert all(torch.equal(a, b) for a, b in zip(out, want))
    for want_dx in (False, True):
        Xg = X.clone().requires_grad_(want_dx)
        grads = []
        for scale in (1.0, 1.0, 8.0):
            m.zero_grad()
            o = m(Xg, ei, ew, H, C)
            loss = (o[0].square().mean() + o[2].mean()) * scale
            _, n = _launches(lambda: loss.backward())
            assert n == 3 + Lg + (1 if (mx or want_dx) else 0) + 2
            grads.append([p.grad.clone() for p in m.parameters()] + ([Xg.grad.clone()] if want_dx else []))
            if want_dx:
                Xg.grad = None
        assert all(torch.equal(a, b) for a, b in zip(grads[0], grads[1]))
        assert all(torch.equal(a * 8, b) for a, b in zip(grads[0], grads[2]))


@pytest.mark.parametrize("C,Ll,dtype,conv,lstm", [(20, 1, torch.float32, True, False), (8, 2, torch.float32, True, False),
                                                  (8, 1, torch.float64, False, False), (8, 1, torch.float32, True, True)])
def test_routes(C, Ll, dtype, conv, lstm):
    """C in 17..32 or two LSTM layers: the row-split convolution feeds the module's cuDNN LSTM; float64: op for op."""
    torch.manual_seed(0)
    m = DyGrEncoder(C, 2, "mean", 32, Ll).to(DEV).to(dtype)
    ei = _graph_of("random", 200, 1).to(DEV)
    X = torch.randn(200, 6, device=DEV, dtype=dtype)
    before = dict(_lib.path_counters())
    with torch.no_grad():
        h, H, Cc = m(X, ei)
    after = _lib.path_counters()
    assert (after.get("k_ggc_rows_fwd", 0) > before.get("k_ggc_rows_fwd", 0)) is conv
    assert (after.get("k_lstm_rows_fwd", 0) > before.get("k_lstm_rows_fwd", 0)) is lstm
    p64 = _params64(m)
    want = dygrae_step(p64, dict(C=C, Lg=2, aggr="mean", Ho=32, Ll=Ll), X.double().cpu(), ei.cpu(), None)
    for a, b, what in zip((h, H, Cc), want, ("H_tilde", "H", "C")):
        _close(a, b, what, 1e-4)
    assert h.data_ptr() != H.data_ptr()


def test_carried_state_errors():
    m = DyGrEncoder(4, 1, "mean", 32, 1).to(DEV)
    x, ei = torch.randn(1, 3, device=DEV), torch.zeros(2, 0, dtype=torch.int64, device=DEV)
    _, H, C = m(x, ei)
    assert H.shape == (32,)
    with pytest.raises(IndexError):
        m(x, ei, None, H, C)
    m = DyGrEncoder(4, 1, "mean", 32, 2).to(DEV)
    x, ei = torch.randn(5, 3, device=DEV), torch.tensor([[0, 1], [1, 2]], device=DEV)
    _, H, C = m(x, ei)
    with pytest.raises(RuntimeError):
        m(x, ei, None, H, C)
    with pytest.raises(RuntimeError):                       # batched X is not supported by the reference either
        m(torch.randn(2, 5, 3, device=DEV), ei)


def test_cuda_graph_tutorial_epoch():
    c = load(GOLDEN)["cases"]["tutorial"]
    ei, ew, X, Y = chickenpox_train_split()
    m = model_for(c, DEV)
    X, Y, ei, ew = X.to(DEV), Y.to(DEV), ei.to(DEV), ew.to(DEV)
    with torch.no_grad():
        want, _ = run(m, X, Y, ei, ew)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        run(m, X, Y, ei, ew)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.no_grad():
        got, _ = run(m, X, Y, ei, ew)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_abi_errors():
    ei, ew, _, _ = chickenpox_train_split()
    L = _lib.lib()
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 20, "sym")
    gp = GatedPlan(ei.to(DEV), ew.to(DEV), 20, "max")
    assert L.stmp_ggc_rows_supported(gp.handle, 3, 4, 32) == 1
    assert L.stmp_ggc_rows_supported(gp.handle, 1, 33, 33) == 0
    assert L.stmp_ggc_rows_supported(gp.handle, 1, 5, 4) == 0
    assert L.stmp_ggc_rows_supported(gp.handle, 0, 4, 4) == 0
    assert L.stmp_ggc_rows_supported(cheb.handle, 1, 4, 4) == 0
    assert L.stmp_lstm_rows_supported(gp.handle, _lib.LSTM_GCONV, 0, 16, 32) == 1
    assert L.stmp_lstm_rows_supported(gp.handle, _lib.LSTM_GCONV, 0, 16, 64) == 1
    buf = torch.zeros(1 << 20, device=DEV)
    p = _lib.ptr(buf)
    fwd = lambda plan, L_, cin, C: L.stmp_ggc_rows_fwd(plan, L_, cin, C, p, p, p, p, p, p, p, p, None, None)
    assert fwd(cheb.handle, 1, 4, 4) == _lib.STMP_EINVAL
    assert fwd(None, 1, 4, 4) == _lib.STMP_EINVAL
    assert fwd(gp.handle, 1, 5, 4) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_ggc_rows_fwd(gp.handle, 1, 4, 4, p, p, p, p, p, p, None, p, None, None) == _lib.STMP_EINVAL
    assert L.stmp_ggc_rows_bwd(gp.handle, 1, 4, 4, p, None, p, p, p, p, p, p, None, None) == _lib.STMP_EINVAL
    assert L.stmp_ggc_rows_wgrad(gp.handle, 1, 4, p, p, p, p, p, p, p, p, None, None) == _lib.STMP_EINVAL
    assert L.stmp_ggc_rows_wgrad_workspace_bytes(2, 32) > 0 and L.stmp_ggc_rows_wgrad_workspace_bytes(2, 33) == 0
    assert L.stmp_ggc_rows_scratch_bytes(gp.handle, 8) == 4 * 20 * 8 * 4
    torch.cuda.synchronize()
