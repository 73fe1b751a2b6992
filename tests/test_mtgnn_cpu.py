"""MTGNN without a GPU: the op-for-op restatement against the unmodified reference in float64 (every golden case: two training
steps with Adam, every gradient, the eval call), the state_dict keys and seeded initialisation against the reference's, the sparse
backward's decomposition (mtgnn.cu's algebra written in float64 torch) against autograd of the dense reference algebra, the
reference's k > N error, the routing predicate and the refusal of CPU tensors."""
import pytest
import torch

from mtgnn_seq import CASES, build, model_for, run
from oracle import refload
from pytorch_geometric_temporal_b200.nn.attention import MTGNN, GraphConstructor, MixProp
from pytorch_geometric_temporal_b200.nn.attention import mtgnn as M

D = torch.float64


def _ref_module():
    if not refload.available():
        pytest.skip("reference tree not present")
    return refload.load("nn.attention.mtgnn")


@pytest.fixture
def on_cpu(monkeypatch):
    """Lift the modules' CUDA-only check so the op-for-op route runs on CPU tensors."""
    monkeypatch.setattr(M, "_require_cuda", lambda t, name: None)


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_reference(name, on_cpu):
    """The whole model, op for op on CPU in float64, against the reference: every output, loss and gradient of both Adam steps and
    the eval output.  The convolutions run as unfold + einsum, which sums in another order than conv2d, so agreement is to 1e-10 of
    each tensor's scale."""
    ref_mod = _ref_module()
    c = CASES[name]
    old = torch.get_default_dtype()
    torch.set_default_dtype(D)
    try:
        want = run(model_for(c, ref_mod.MTGNN, "cpu", D), c, "cpu", D)
        got = run(model_for(c, MTGNN, "cpu", D), c, "cpu", D)
    finally:
        torch.set_default_dtype(old)
    assert set(got) == set(want)
    for k in want:
        assert got[k].shape == want[k].shape, k
        tol = 1e-10 * float(want[k].abs().max())
        assert float((got[k] - want[k]).abs().max()) <= tol, (k, float((got[k] - want[k]).abs().max()), tol)


@pytest.mark.parametrize("name", ["idx", "fe", "nogcn_dil2", "seq24"])
def test_state_dict_and_seeded_init_match_reference(name):
    ref_mod = _ref_module()
    c = CASES[name]
    torch.manual_seed(5)
    want = build(ref_mod.MTGNN, c).state_dict()
    torch.manual_seed(5)
    got_m = build(MTGNN, c)
    got = got_m.state_dict()
    assert list(got) == list(want)
    for k in want:
        assert torch.equal(got[k], want[k]), k
    assert not any(k.endswith("_idx") for k in got)        # a plain attribute, as in the reference
    torch.manual_seed(6)
    a = ref_mod.MixProp(8, 4, 2, 0.3, 0.05).state_dict()
    torch.manual_seed(6)
    b = MixProp(8, 4, 2, 0.3, 0.05).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    torch.manual_seed(7)
    a = ref_mod.GraphConstructor(30, 5, 6, 3.0).state_dict()
    torch.manual_seed(7)
    b = GraphConstructor(30, 5, 6, 3.0).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_graph_constructor_and_mixprop_match_reference(on_cpu):
    ref_mod = _ref_module()
    old = torch.get_default_dtype()
    torch.set_default_dtype(D)               # the reference builds its mask in the default dtype
    try:
        _graph_constructor_and_mixprop(ref_mod)
    finally:
        torch.set_default_dtype(old)


def _graph_constructor_and_mixprop(ref_mod):
    torch.manual_seed(8)
    ref = ref_mod.GraphConstructor(40, 6, 5, 3.0).double()
    ours = GraphConstructor(40, 6, 5, 3.0).double()
    ours.load_state_dict(ref.state_dict())
    idx = torch.randperm(40)
    assert torch.equal(ours(idx), ref(idx))
    X = torch.randn(2, 3, 40, 5, dtype=D)
    A = ref(idx).detach()
    mp_ref = ref_mod.MixProp(3, 4, 3, 0.3, 0.1).double()
    mp = MixProp(3, 4, 3, 0.3, 0.1).double()
    mp.load_state_dict(mp_ref.state_dict())
    assert torch.allclose(mp(X, A), mp_ref(X, A), rtol=0, atol=1e-12)


def test_k_above_n_raises_reference_error():
    g = GraphConstructor(5, 8, 4, 3.0)
    with pytest.raises(RuntimeError, match="selected index k out of range"):
        g.sparse(torch.arange(5), None, False)


def test_modules_refuse_cpu_tensors():
    m = MTGNN(**dict(CASES["plain"]["model"], num_nodes=10, subgraph_size=3))
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.randn(2, 2, 10, 12))


def test_routing_predicate(monkeypatch):
    monkeypatch.setattr(M.ops, "mtgnn_supported", lambda *a: True)
    f32, f64 = torch.float32, torch.float64
    args = (207, 20, 40, 32, 2, 4, 19)
    assert M.fused_route(f32, True, *args, True, False, True)
    assert M.fused_route(f32, True, *args, True, True, True)
    assert not M.fused_route(f32, True, *args, True, True, False)         # training with fused_training = False
    assert M.fused_route(f32, True, *args, True, False, False)            # inference ignores fused_training
    assert not M.fused_route(f64, True, *args, True, False, True)
    assert not M.fused_route(f32, False, *args, True, False, True)
    assert not M.fused_route(f32, True, *args, False, False, True)         # gcn_true = False
    monkeypatch.setattr(M.ops, "mtgnn_supported", lambda *a: False)
    assert not M.fused_route(f32, True, *args, True, False, True)


# ---- mtgnn.cu's algebra in float64 torch ------------------------------------------------------------------------------------------
def _dense_reference(m1, m2, X, W1, W2, alpha, talpha, k, depth):
    """The reference's algebra: graph, both MixProps and their MLPs (weights (C_out, (depth + 1) C))."""
    a = m1 @ m2.T - m2 @ m1.T
    A = torch.relu(torch.tanh(talpha * a))
    mask = torch.zeros_like(A).scatter_(1, A.topk(k, 1).indices, 1.0)
    A = A * mask
    out = 0
    for Aop, W in ((A, W1), (A.T, W2)):
        Ah = Aop + torch.eye(A.shape[0], dtype=D)
        Ah = Ah / Ah.sum(1).view(-1, 1)
        H, hs = X, [X]
        for _ in range(depth):
            H = alpha * X + (1 - alpha) * torch.einsum("ncwl,vw->ncvl", H, Ah)
            hs.append(H)
        out = out + torch.einsum("oc,bcnt->bont", W, torch.cat(hs, 1))
    return out


def _sparse_decomposition(m1, m2, X, W1, W2, alpha, talpha, k, depth, gy):
    """dX, dM1, dM2 as the kernels compute them: the hop chains over the top-k pattern, the adjoint chains, the sampled products on the
    pattern and diagonals, both normalisations' backward, the mask / relu / tanh, then dM1 = (dz - dz^T) M2 and dM2 = (dz^T - dz) M1."""
    n, C = m1.shape[0], X.shape[1]
    z = m1 @ m2.T - m2 @ m1.T
    Araw = torch.relu(torch.tanh(talpha * z))
    P = torch.zeros_like(Araw, dtype=torch.bool).scatter_(1, Araw.topk(k, 1).indices, True) & (Araw > 0)   # zeros dropped
    a = torch.where(P, Araw, 0.0)
    d1, d2 = 1 + a.sum(1), 1 + a.sum(0)
    V1, V2 = a / d1[:, None], (a / d2[None, :])           # V2[i, j] = entry (j, i) of operator 2, stored at (i, j)
    S = [torch.diag(1 / d1) + V1, torch.diag(1 / d2) + V2.T]
    Ws = [W1, W2]
    gx = sum(torch.einsum("oc,bont->bcnt", W[:, :C], gy) for W in Ws)
    dS = []
    for o in range(2):
        Hs = [X]
        for _ in range(depth):
            Hs.append(alpha * X + (1 - alpha) * torch.einsum("vw,bcwt->bcvt", S[o], Hs[-1]))
        G = [None] + [torch.einsum("oc,bont->bcnt", Ws[o][:, (q + 1) * C:(q + 2) * C], gy) for q in range(depth)]
        dSo = torch.zeros(n, n, dtype=D)
        for q in range(depth, 0, -1):
            gx = gx + alpha * G[q]
            back = (1 - alpha) * torch.einsum("vw,bcvt->bcwt", S[o], G[q])
            dSo = dSo + (1 - alpha) * torch.einsum("bcvt,bcwt->vw", G[q], Hs[q - 1])
            if q == 1:
                gx = gx + back
            else:
                G[q - 1] = G[q - 1] + back
        dS.append(dSo)
    dv1 = torch.where(P, dS[0], 0.0)
    dv2 = torch.where(P, dS[1].T, 0.0)                     # at the (i, j) position of A
    ddiag1, ddiag2 = dS[0].diagonal(), dS[1].diagonal()
    dd1 = -((dv1 * V1).sum(1) + ddiag1 / d1) / d1
    dd2 = -((dv2 * V2).sum(0) + ddiag2 / d2) / d2
    da = torch.where(P, dv1 / d1[:, None] + dv2 / d2[None, :] + dd1[:, None] + dd2[None, :], 0.0)
    dz = da * talpha * (1 - a * a)
    return gx, (dz - dz.T) @ m2, (dz.T - dz) @ m1


@pytest.mark.parametrize("n,k,depth,dim", [(12, 4, 1, 3), (17, 5, 2, 4), (9, 9, 3, 2), (20, 1, 4, 5)])
def test_sparse_backward_decomposition_matches_autograd(n, k, depth, dim):
    g = torch.Generator().manual_seed(n * 100 + k)
    B, C, T, Co, alpha, talpha = 2, 3, 4, 5, 0.05, 3.0
    m1 = (0.3 * torch.randn(n, dim, generator=g, dtype=D)).requires_grad_(True)
    m2 = (0.3 * torch.randn(n, dim, generator=g, dtype=D)).requires_grad_(True)
    X = torch.randn(B, C, n, T, generator=g, dtype=D, requires_grad=True)
    W1 = torch.randn(Co, (depth + 1) * C, generator=g, dtype=D)
    W2 = torch.randn(Co, (depth + 1) * C, generator=g, dtype=D)
    gy = torch.randn(B, Co, n, T, generator=g, dtype=D)
    out = _dense_reference(m1, m2, X, W1, W2, alpha, talpha, k, depth)
    want = torch.autograd.grad(out, (X, m1, m2), gy)
    got = _sparse_decomposition(m1.detach(), m2.detach(), X.detach(), W1, W2, alpha, talpha, k, depth, gy)
    for w, h in zip(want, got):
        assert torch.allclose(h, w, rtol=1e-10, atol=1e-11 * float(w.abs().max())), float((h - w).abs().max())


def _no_launch(*a, **k):
    raise AssertionError("a k_mtgnn_* entry was called")


def test_node_count_mismatch_raises_before_any_launch(on_cpu, monkeypatch):
    """idx selects 100 of 207 nodes while X keeps all 207: the learned graph has 100 nodes.  The model must not hand that graph to the
    kernels (they trust N): the call runs op for op, where the reference's einsum raises its size error, and no kernel entry runs."""
    monkeypatch.setattr(M, "fused_route", lambda *a: True)          # every other condition of the fused route holds
    for name in ("mtgnn_graph", "mtgnn_graph_fwd", "mtgnn_graph_dense", "mtgnn_mixprop", "mtgnn_prop_fwd"):
        monkeypatch.setattr(M.ops, name, _no_launch)
    m = MTGNN(**dict(CASES["plain"]["model"], num_nodes=207))
    X = torch.randn(2, 2, 207, 12)
    assert not m._fused(X, 100, 20, 40) and m._fused(X, 207, 20, 40)
    with pytest.raises(RuntimeError, match="einsum"):
        m(X, idx=torch.randperm(207)[:100])
    p = MTGNN(**dict(CASES["plain"]["model"], num_nodes=207, build_adj=False))
    with pytest.raises(RuntimeError, match="einsum"):
        p(X, (torch.rand(100, 100) < 0.1).float())


def test_layer_refuses_a_graph_of_another_node_count(on_cpu, monkeypatch):
    monkeypatch.setattr(M.ops, "mtgnn_mixprop", _no_launch)
    layer = M.MTGNNLayer(1, 1, 7, 1, 32, 32, 64, [2, 3, 6, 7], 1, True, True, 12, 19, 0.0, 2, 207, 0.05)
    g = M._Graph(torch.zeros(2 * 100 * 20 + 200), torch.zeros(3 * 100 * 20 + 201, dtype=torch.int32), 100, 20)
    with pytest.raises(RuntimeError, match="graph has 100 nodes, X has 207"):
        layer(torch.randn(2, 32, 207, 19), torch.zeros(2, 64, 207, 1), g, torch.arange(207), False)


def test_propagation_wrapper_checks_the_graph_buffers():
    """ops.mtgnn_prop_fwd checks the pattern and values against X's node count and the row width before anything else."""
    from pytorch_geometric_temporal_b200 import ops
    n, w = 30, 5
    pattern, vals = torch.zeros(3 * n * w + 2 * n + 1, dtype=torch.int32), torch.zeros(2 * n * w + 2 * n)
    x = torch.randn(2, 3, n + 1, 4)
    with pytest.raises(RuntimeError, match="pattern has"):
        ops.mtgnn_prop_fwd(x, pattern, vals, w, 2, 0.05)
    with pytest.raises(RuntimeError, match="values has"):
        ops.mtgnn_prop_fwd(torch.randn(2, 3, n, 4), pattern, vals[:-1], w, 2, 0.05)
    with pytest.raises(RuntimeError, match="int32"):
        ops.mtgnn_prop_fwd(torch.randn(2, 3, n, 4), pattern.long(), vals, w, 2, 0.05)
    with pytest.raises(RuntimeError, match="CUDA only"):       # sizes right: the next check is the device
        ops.mtgnn_prop_fwd(torch.randn(2, 3, n, 4), pattern, vals, w, 2, 0.05)
