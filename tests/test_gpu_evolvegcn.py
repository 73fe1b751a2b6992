"""EvolveGCNO / EvolveGCNH on the H100: every golden case on the row-split kernels and op for op against the float64 oracle (held to the
reference's fingerprints by tests/test_evolvegcn_cpu.py), the envelope against float64, adversarial graphs, TopK ties, bit-reproducible
and loss-scale-equivariant gradients with training forwards equal to inference, exact launch counts, a chain of calls with the weight reset
or detached, retain_graph, CUDA-graph replay and the ABI's errors.  Tolerances are test_gpu_dygrae.py's (_close: the largest error over the
float64 tensor's largest magnitude, 2e-4 for outputs, 1e-3 for gradients)."""
import os

import pytest
import torch

from evolvegcn_seq import egcn_step, graph_of, load, model_for, oracle_run, run
from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.nn.recurrent import EvolveGCNH, EvolveGCNO
from pytorch_geometric_temporal_b200.nn.recurrent.evolvegcn import topk_size
from pytorch_geometric_temporal_b200.plan import GatedPlan, GraphPlan
from test_gpu_rows_envelope import _counted

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EG = ("k_egcn_fwd", "k_egcn_score", "k_egcn_fwd_topk", "k_egcn_bwd_rows", "k_egcn_wgrad", "k_egcn_wgrad_topk")


@pytest.fixture(autouse=True)
def _fp32():
    """cuDNN's GRU and cuBLAS in full fp32 on the op-for-op route."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _close(got, want, what, rtol=2e-4, scale=None):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = (float(want.abs().max()) if scale is None else scale) + 1e-30
    err = float((got - want).abs().max()) / scale
    assert err <= rtol, (what, err)


def _ran(c):
    return {k: v for k, v in c.items() if k in EG}


def _launches(topk, train, want_dx=True):
    want = {"k_egcn_score": 1, "k_egcn_fwd_topk": 1} if topk else {"k_egcn_fwd": 1}
    if train:
        want.update({"k_egcn_bwd_rows": 1, "k_egcn_wgrad_topk" if topk else "k_egcn_wgrad": 1})
    return want


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_golden_cases(name, fused):
    c = load(GOLDEN)["cases"][name]
    ei, ew, X, Y = graph_of(c, GOLDEN)
    outs64, cost64, leaves = oracle_run(c, X, Y, ei, ew, c["epochs"])
    m = model_for(c, DEV, fused)
    with _counted() as cnt:
        outs, cost = run(m, X.to(DEV), Y.to(DEV), ei.to(DEV), None if ew is None else ew.to(DEV), c["epochs"], retain=True)
    steps = c["epochs"] * X.shape[0]
    assert _ran(cnt) == ({k: steps * v for k, v in _launches(c["kind"] == "H", True).items()} if fused else {}), cnt
    assert abs(float(cost.detach()) - float(cost64.detach())) <= 1e-5 * abs(float(cost64.detach()))
    _close(outs, outs64, "out")
    for k, p in m.named_parameters():
        _close(p.grad, leaves[k].grad, k, 1e-3)


def _graph(kind, n, seed):
    """edge_index and positive weights of a named geometry: random (with duplicates and self loops), "holes" (rows without in-edges and
    isolated nodes), "E0" (no edge)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "E0":
        return torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0)
    e = 3 * n
    src, dst = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
    if kind == "holes":
        dst = dst % max(1, n // 2)
        src = src % max(1, n - 2)
    ei = torch.stack([src, dst])
    ei = torch.cat([ei, ei[:, :e // 5], torch.stack([src[:3], src[:3]])], 1)
    return ei, torch.rand(ei.size(1), generator=g) * 2


def _nodes_for(C, n):
    """A num_of_nodes >= n whose ratio C / num_of_nodes keeps exactly C of n nodes in float32 and float64 (N itself, unless ceil(ratio N)
    rounds up to C + 1)."""
    nodes = n
    while any(topk_size(C / nodes, n, d) != C for d in (torch.float32, torch.float64)):
        nodes += 1
    return nodes


def _case(kind, C, n, ew_kind, seed, flags=None):
    """(model, c, X, ei, ew) with N(0, 0.5) parameters."""
    flags = flags or dict(improved=False, normalize=True, add_self_loops=True)
    torch.manual_seed(seed)
    nodes = _nodes_for(C, n) if kind == "H" else n
    m = (EvolveGCNH(nodes, C, **flags) if kind == "H" else EvolveGCNO(C, **flags))
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.5)
    c = dict(kind=kind, C=C, nodes=nodes, normalize=flags["normalize"], improved=flags["improved"], loops=flags["add_self_loops"])
    ei, ew = _graph("holes" if seed % 3 == 1 else "random", n, seed)
    if ew_kind is None:
        ew = None
    elif ew_kind == "signed":                 # gcn_norm of a negative degree is NaN (PyG's too): signed weights on the raw operator only
        ew = ew - 1 if not flags["normalize"] else ew
        ew[::5] = 0.0
    X = torch.randn(n, C, generator=torch.Generator().manual_seed(seed))
    return m.to(DEV), c, X, ei, ew


def _check_steps(m, c, X, ei, ew, steps=2, want_dx=True):
    """`steps` calls with the weight carried, then one backward, against egcn_step in float64: outputs, dX and every parameter's gradient;
    the launches of each call asserted."""
    p64 = {k: v.detach().double().cpu().requires_grad_(True) for k, v in m.named_parameters()}
    x64 = X.double().requires_grad_(want_dx)
    ew64 = None if ew is None else ew.double()
    W, o64 = None, []
    for _ in range(steps):
        o, W = egcn_step(p64, c, W, x64, ei, ew64)
        o64.append(o)
    coef = [torch.randn(o.shape, generator=torch.Generator().manual_seed(i), dtype=torch.float64) for i, o in enumerate(o64)]
    sum((a * b).sum() for a, b in zip(o64, coef)).backward()
    xd = X.to(DEV).requires_grad_(want_dx)
    eid, ewd = ei.to(DEV), None if ew is None else ew.to(DEV)
    m.weight = None
    m.zero_grad(set_to_none=True)
    with _counted() as cnt:
        outs = [m(xd, eid, ewd) for _ in range(steps)]
        sum((a * b.float().to(DEV)).sum() for a, b in zip(outs, coef)).backward()
    assert _ran(cnt) == {k: steps * v for k, v in _launches(c["kind"] == "H", True).items()}, cnt
    for a, b in zip(outs, o64):
        _close(a, b, "out")
    # At C = 1 the score tanh(x p / |p|) does not depend on |p|: the pooling weight's gradient is exactly 0 and only rounding is left of
    # it, so it is measured against the model's largest parameter gradient.
    top = max(float(g.grad.abs().max()) for g in p64.values())
    for k, q in m.named_parameters():
        _close(q.grad, p64[k].grad, k, 1e-3, top if (c["C"] == 1 and k == "pooling_layer.select.weight") else None)
    if want_dx:
        _close(xd.grad, x64.grad, "dX", 1e-3)


@pytest.mark.parametrize("kind", ["O", "H"])
@pytest.mark.parametrize("C", [1, 4, 8, 14, 16, 31, 32])
@pytest.mark.parametrize("n", [1, 3, 16, 17, 33, 4225])
def test_envelope_against_float64(kind, C, n):
    """C in 1..32 on 1 node up through 16-row tiles to 4 225 (where the grid stride starts); -H needs N >= C and k = C, so it runs with
    num_of_nodes = N where N >= C; -O also at N < C."""
    if kind == "H" and n < C:
        pytest.skip("-H selects C of N nodes")
    seed = 100 * C + n
    m, c, X, ei, ew = _case(kind, C, n, ("pos", None, "signed")[seed % 3], seed)
    _check_steps(m, c, X, ei, ew, want_dx=seed % 2 == 0)


@pytest.mark.parametrize("kind", ["O", "H"])
def test_50000_nodes_against_float64(kind):
    m, c, X, ei, ew = _case(kind, 32, 50000, "pos", 7)
    _check_steps(m, c, X, ei, ew, steps=1)


@pytest.mark.parametrize("flags", [dict(improved=True, normalize=True, add_self_loops=True),
                                   dict(improved=False, normalize=True, add_self_loops=False),
                                   dict(improved=False, normalize=False, add_self_loops=True)])
@pytest.mark.parametrize("kind", ["O", "H"])
def test_flags_and_adversarial_graphs(kind, flags):
    """improved, no self loops and the raw edge weights on graphs with duplicates, self loops, rows without in-edges, isolated nodes and
    zero and negative weights; and on a graph without edges."""
    for seed, ewk in ((1, "signed"), (4, None), (2, "pos")):      # signed: zero and (normalize=False) negative weights
        m, c, X, ei, ew = _case(kind, 8, 97, ewk, seed, flags)
        _check_steps(m, c, X, ei, ew)
    m, c, X, _, _ = _case(kind, 8, 40, None, 3, flags)
    ei, ew = _graph("E0", 40, 0)
    _check_steps(m, c, X, ei, ew)


@pytest.mark.parametrize("n", [40, 5000])
def test_topk_ties_select_the_lower_index(n):
    """Many nodes share the same X row (exact score ties): the selection is the lower indices first, as the stable sort's; checked
    against the op-for-op route's perm and against float64."""
    C = 8
    m, c, X, ei, ew = _case("H", C, n, "pos", 5)
    X[:] = X[0]
    X[n // 2:] = X[1]
    X[n - 3] = X[2]
    from pytorch_geometric_temporal_b200 import ops
    from evolvegcn_seq import topk_pool
    plan = m._plan(ei.to(DEV), ew.to(DEV), n)
    r = m.recurrent_layer
    _, _, perm, score, _ = ops.evolvegcn_rows_fwd(plan, X.to(DEV), m.initial_weight[0], r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0,
                                                  r.bias_hh_l0, m.pooling_layer.select.weight.view(-1))
    _, want, s = topk_pool(X.double(), m.pooling_layer.select.weight.detach().double().cpu(), C / n)
    assert perm.long().cpu().tolist() == want.tolist()
    _check_steps(m, c, X, ei, ew)


@pytest.mark.parametrize("kind", ["O", "H"])
def test_reproducible_and_training_equals_inference(kind):
    m, c, X, ei, ew = _case(kind, 16, 3000, "pos", 9)
    X, ei, ew = X.to(DEV), ei.to(DEV), ew.to(DEV)
    with torch.no_grad():
        m.weight = None
        want = [m(X, ei, ew) for _ in range(3)]
        m.weight = None
        again = [m(X, ei, ew) for _ in range(3)]
    assert all(torch.equal(a, b) for a, b in zip(want, again))
    grads = []
    for scale in (1.0, 1.0, 8.0):
        m.weight = None
        m.zero_grad()
        Xg = X.clone().requires_grad_(True)
        outs = [m(Xg, ei, ew) for _ in range(3)]
        assert all(torch.equal(a.detach(), b) for a, b in zip(outs, want))
        (sum(o.square().mean() for o in outs) * scale).backward()
        grads.append([p.grad.clone() for p in m.parameters()] + [Xg.grad.clone()])
    assert all(torch.equal(a, b) for a, b in zip(grads[0], grads[1]))
    assert all(torch.equal(a * 8, b) for a, b in zip(grads[0], grads[2]))


@pytest.mark.parametrize("kind", ["O", "H"])
def test_chain_reset_detach_and_retain_graph(kind):
    """Five calls where the weight is detached after the second and reset to None after the fourth, fused against op for op; then a
    second backward through the retained graph gives the same gradients."""
    res = {}
    for fused in (True, False):
        m, c, X, ei, ew = _case(kind, 8, 200, "pos", 12)
        m.fused_training = fused
        X, ei, ew = X.to(DEV), ei.to(DEV), ew.to(DEV)
        loss = 0
        for t in range(5):
            loss = loss + m(X * (1 + 0.1 * t), ei, ew).square().mean()
            if t == 1:
                m.weight = m.weight.detach()
            if t == 3:
                m.weight = None
        loss.backward(retain_graph=True)
        g1 = [p.grad.clone() for p in m.parameters()]
        m.zero_grad()
        loss.backward()
        g2 = [p.grad.clone() for p in m.parameters()]
        if fused:
            assert all(torch.equal(a, b) for a, b in zip(g1, g2))
        res[fused] = (float(loss), g1)
    assert abs(res[True][0] - res[False][0]) <= 1e-5 * abs(res[False][0])
    for a, b in zip(res[True][1], res[False][1]):
        _close(a, b, "grad", 1e-3)


@pytest.mark.parametrize("kind", ["O", "H"])
def test_cuda_graph_no_grad_call(kind):
    m, c, X, ei, ew = _case(kind, 32, 50000, "pos", 2)
    X, ei, ew = X.to(DEV), ei.to(DEV), ew.to(DEV)
    with torch.no_grad():
        m.weight = None
        want = m(X, ei, ew)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m.weight = None
            m(X, ei, ew)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        m.weight = None
        with torch.cuda.graph(graph):
            got = m(X, ei, ew)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_routes():
    """float64, C > 32 and a gradient into edge_weight run op for op (no row-split launch) and match float64."""
    for kind, C, dtype, ew_grad in (("O", 8, torch.float64, False), ("H", 40, torch.float32, False), ("O", 8, torch.float32, True)):
        m, c, X, ei, ew = _case(kind, C, 120, "pos", 3)
        m = m.to(dtype)
        ewd = ew.to(DEV, dtype).requires_grad_(ew_grad)
        with _counted() as cnt:
            out = m(X.to(DEV, dtype), ei.to(DEV), ewd)
            out.sum().backward()
        assert _ran(cnt) == {}, cnt
        p64 = {k: v.detach().double().cpu() for k, v in m.named_parameters()}
        _close(out, egcn_step(p64, c, None, X.double(), ei, ew.double())[0], "out", 1e-4)


def test_abi_errors():
    ei, ew = _graph("random", 20, 1)
    ei, ew = ei.to(DEV), ew.to(DEV)
    L = _lib.lib()
    gcn = GraphPlan(_lib.FLAVOR_GCN, ei, ew, 20, None)
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei, ew, 20, "sym")
    mean = GatedPlan(ei, ew, 20, "mean")
    add = GatedPlan(ei, ew, 20, "add")
    assert L.stmp_evolvegcn_rows_supported(gcn.handle, 32) == 1 and L.stmp_evolvegcn_rows_supported(add.handle, 1) == 1
    assert L.stmp_evolvegcn_rows_supported(gcn.handle, 33) == 0 and L.stmp_evolvegcn_rows_supported(gcn.handle, 0) == 0
    assert L.stmp_evolvegcn_rows_supported(mean.handle, 4) == 0 and L.stmp_evolvegcn_rows_supported(cheb.handle, 4) == 0
    buf = torch.zeros(1 << 20, device=DEV)
    p = _lib.ptr(buf)
    fwd = lambda plan, C, *tail: L.stmp_evolvegcn_rows_fwd(plan, C, p, p, p, p, p, p, *tail)
    assert fwd(cheb.handle, 4, None, None, p, p, None, None, None, None) == _lib.STMP_EINVAL
    assert fwd(None, 4, None, None, p, p, None, None, None, None) == _lib.STMP_EINVAL
    assert fwd(mean.handle, 4, None, None, p, p, None, None, None, None) == _lib.STMP_EUNSUPPORTED
    assert fwd(gcn.handle, 33, None, None, p, p, None, None, None, None) == _lib.STMP_EUNSUPPORTED
    assert fwd(gcn.handle, 4, None, None, None, p, None, None, None, None) == _lib.STMP_EINVAL
    assert fwd(gcn.handle, 4, p, None, p, p, p, p, None, None) == _lib.STMP_EINVAL                  # -H without scratch
    assert fwd(gcn.handle, 21, p, p, p, p, p, p, None, None) == _lib.STMP_EUNSUPPORTED               # -H on fewer nodes than C
    assert fwd(gcn.handle, 4, None, None, p, ctypes_misaligned(buf), None, None, None, None) == _lib.STMP_ESHAPE
    assert L.stmp_evolvegcn_rows_bwd(gcn.handle, 4, p, None, p, p, None, None) == _lib.STMP_EINVAL
    assert L.stmp_evolvegcn_rows_wgrad(gcn.handle, 4, p, None, p, p, p, p, p, p, p, None, None, p, p, p, p, p, None, None,
                                       None) == _lib.STMP_EINVAL                                     # -H without perm, score and dp
    assert L.stmp_evolvegcn_rows_wgrad(gcn.handle, 4, None, *([p] * 16), None, None) == _lib.STMP_EINVAL
    assert L.stmp_evolvegcn_rows_workspace_bytes(gcn.handle, 33) == 0 and L.stmp_evolvegcn_rows_workspace_bytes(gcn.handle, 4) > 0
    assert L.stmp_evolvegcn_rows_scratch_bytes(gcn.handle, 4) >= 4 * 20
    torch.cuda.synchronize()


def ctypes_misaligned(buf):
    import ctypes
    return ctypes.c_void_p(buf.data_ptr() + 2)
