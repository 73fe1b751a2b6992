"""BatchedDCRNN(cin, 32, 2) on graphs larger than one SM: the row-split kernels (`stmp_dcrnn_rows_*`, DESIGN §4k).  The PEMS-BAY shape
against the unmodified reference (tests/golden/make_goldens_dcrnn_rows.py); the forward against the float64 oracle across the envelope
(the smallest graph the one-SM kernels refuse, PEMS-BAY, random graphs with hubs, a 50 000-node graph; every cin, B in {1, 3, 64}, T in
{1, 2, 12}); the reference's non-finite pattern on zero-degree nodes; fused training against autograd through the tiled path;
bit-identity of the training forward, determinism and loss-scale equivariance of the backward; index batching and empty calls; a
PeMS-like size whose weight-gradient operands pass 2^31 bytes; a captured training step; routing, launch budgets and the C ABI's errors."""
import contextlib
import ctypes
import gzip
import os

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200 import distributed as D
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN, BatchedDCRNN
from pytorch_geometric_temporal_b200.plan import GraphPlan

pytestmark = pytest.mark.gpu
DEV = "cuda"
FWD = ("k_dcrnn_rows_fwd_a", "k_dcrnn_rows_fwd_b")
BWD = ("k_dcrnn_rows_bwd_start", "k_dcrnn_rows_bwd_b", "k_dcrnn_rows_bwd_c", "k_dcrnn_rows_bwd_x")
ROWS = FWD + BWD


@contextlib.contextmanager
def _counted():
    """Yields a dict that, after the block, holds {kernel: launches during the block}."""
    c0, delta = _lib.path_counters(), {}
    yield delta
    c1 = _lib.path_counters()
    delta.update({k: v - c0.get(k, 0) for k, v in c1.items() if v != c0.get(k, 0)})


@contextlib.contextmanager
def _float64():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)       # the oracle's zeros / scatter buffers
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def _rows_only(c):
    """the launches of the row-split kernels and of the tiled path's SpMM in a _counted() delta"""
    return {k: v for k, v in c.items() if k in ROWS or k == "k_spmm"}


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _grad_close(got, ref):
    _close(got, ref, 1e-3, 1e-3 * max(ref.abs().max().item(), 1e-12))


def _graph(n, deg, seed, hubs=False):
    """Random directed graph plus a ring (every node has in- and out-degree >= 1, so DConv stays finite); with `hubs`, node 0 gets
    400 in-edges and node 1 400 out-edges (the one-SM kernels' rows are far shorter)."""
    g = torch.Generator().manual_seed(seed)
    src, dst = torch.randint(0, n, (deg * n,), generator=g), torch.randint(0, n, (deg * n,), generator=g)
    ring = torch.arange(n)
    src, dst = torch.cat([src, ring]), torch.cat([dst, (ring + 1) % n])
    if hubs:
        pick = torch.randperm(n - 2, generator=g)[:400] + 2
        src, dst = torch.cat([src, pick, torch.ones(400, dtype=torch.long)]), torch.cat([dst, torch.zeros(400, dtype=torch.long), pick])
    ei = torch.unique(torch.stack([src, dst]), dim=1)
    ei = ei[:, ei[0] != ei[1]]
    return ei.to(DEV), (torch.rand(ei.size(1), generator=g) + 0.1).to(DEV)


def _model(cin, seed, bias=True):
    torch.manual_seed(seed)
    m = BatchedDCRNN(cin, 32, 2, bias=bias)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith(".bias"):
                p.normal_(0, 0.1)
    return m.to(DEV)


def _train(m, X, ei, ew, w, x_grad=True):
    X = X.clone().requires_grad_(x_grad)
    m.zero_grad(set_to_none=True)
    out = m(X, ei, ew)
    (out * w).sum().backward()
    return [out.detach(), X.grad] + [p.grad.clone() for p in m.parameters()]


# ---- the golden from the unmodified reference -----------------------------------------------------------------------------------------
def test_pems_bay_golden(golden_dir):
    with gzip.open(os.path.join(golden_dir, "dcrnn_rows_pems_bay.pt.gz"), "rb") as f:
        g = torch.load(f, weights_only=False)                                   # `out` holds the output's steps `out_steps`
    steps = g["out_steps"]
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    m.load_state_dict(g["state"])
    ei, ew, X = g["edge_index"].to(DEV).long(), g["edge_weight"].to(DEV), g["X"].to(DEV)
    T = X.size(1)
    assert not ops.dcrnn_seq_supported(m._plan(ei, ew, 325), 2, 32, 2)
    m._rows_packed()                                                            # the packed weights are built once
    with _counted() as c, torch.no_grad():
        out = m(X, ei, ew)
    assert _rows_only(c) == {"k_dcrnn_rows_fwd_a": T, "k_dcrnn_rows_fwd_b": T - 1}          # 2T - 1 launches, no SpMM
    _close(out[:, steps], g["out"])
    Xl = X.clone().requires_grad_(True)
    with _counted() as c:
        out = m(Xl, ei, ew)
        (out * torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)).sum().backward()
    assert "k_spmm" not in c and c["k_dcrnn_rows_fwd_a"] == T and c["k_dcrnn_rows_bwd_b"] == T - 1 and c["k_dcrnn_rows_bwd_x"] == 1
    _close(out[:, steps], g["out"])
    _grad_close(Xl.grad, g["gX"])
    for k, p in m.named_parameters():
        _grad_close(p.grad, g["grads"][k])


# ---- against the float64 oracle -------------------------------------------------------------------------------------------------------
def _smallest_refused():
    for n in range(200, 400):
        ei, ew = _graph(n, 4, n)
        if not ops.dcrnn_seq_supported(GraphPlan(_lib.FLAVOR_DCONV, ei, ew, n, flags=_lib.DCONV_ALLOW_DUPLICATES), 2, 32, 2):
            return n, ei, ew
    raise AssertionError("no graph up to 400 nodes is refused by the one-SM kernels")


def _graph_case(name):
    if name == "smallest":
        return _smallest_refused()
    if name == "pems_bay":
        ei, ew, _ = synthetic.pems_bay_like(0, 16)
        return 325, torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    if name == "n50000":
        return (50000,) + _graph(50000, 4, 50)
    n = int(name[1:])
    return (n,) + _graph(n, 8, n, hubs=True)


# (graph, cin, B, T): every cin, B in {1, 3, 64}, T in {1, 2, 12}; hubs of 400 in- and out-edges on the 1000..2600-node graphs
CASES = [("smallest", 2, 3, 12), ("pems_bay", 1, 3, 12), ("pems_bay", 2, 64, 2), ("pems_bay", 3, 1, 12), ("pems_bay", 4, 3, 1),
         ("h1000", 1, 64, 2), ("h1389", 2, 3, 12), ("h1777", 3, 1, 12), ("h2600", 4, 3, 2), ("h2011", 2, 64, 1), ("n50000", 2, 2, 3)]


@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_forward_vs_float64_oracle(case):
    """Criterion: at most 4x the error of the same oracle in float32, plus 2^-20 of the output's scale."""
    graph, cin, B, T = case
    n, ei, ew = _graph_case(graph)
    m = _model(cin, cin + T)
    X = torch.randn(B, T, n, cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B + T))
    plan = m._plan(ei, ew, n)
    assert not ops.dcrnn_seq_supported(plan, cin, 32, 2) and ops.dcrnn_rows_supported(plan, cin, 32, 2)
    with _counted() as c, torch.no_grad():
        out = m(X, ei, ew)
    assert _rows_only(c) == ({"k_dcrnn_rows_fwd_a": T, "k_dcrnn_rows_fwd_b": T - 1} if T > 1 else {"k_dcrnn_rows_fwd_a": 1})
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    with torch.no_grad():
        ref32 = R.batched_dcrnn(sd, X, ei, ew)
        with _float64():
            ref64 = R.batched_dcrnn({k: v.double() for k, v in sd.items()}, X.double(), ei, ew.double())
    got = out.double()
    assert bool(torch.isfinite(got).all())
    e, e32, scale = float((got - ref64).abs().max()), float((ref32.double() - ref64).abs().max()), float(ref64.abs().max())
    assert e <= 4 * e32 + 2.0 ** -20 * scale, (case, e, e32, scale)


def test_zero_degree_nodes_give_the_reference_non_finite_pattern():
    """A path graph: node 0 has no in-edge, so DConv's 1/deg_in is inf on its out-edge.  inf * 0 = NaN reaches the state at step 0 and
    then spreads one hop per step through P(H*R) -- the reference's pattern, which needs the two-launch form of step 0."""
    n = 300
    ei = torch.stack([torch.arange(n - 1), torch.arange(1, n)]).to(DEV)
    ew = torch.ones(n - 1, device=DEV)
    m = _model(2, 0)
    X = torch.randn(2, 4, n, 2, device=DEV)
    want = R.batched_dcrnn({k: v.detach() for k, v in m.state_dict().items()}, X, ei, ew)
    assert not bool(torch.isfinite(want).all()) and bool(torch.isfinite(want).any())
    for grad in (False, True):
        with _counted() as c, torch.set_grad_enabled(grad):
            got = m(X, ei, ew).detach()
        assert c.get("k_dcrnn_rows_fwd_b") == 4                                # step 0 as two launches
        assert torch.equal(torch.isfinite(got), torch.isfinite(want))
        fin = torch.isfinite(want)
        _close(got[fin], want[fin])


# ---- training: fused against autograd through the tiled path ---------------------------------------------------------------------------
@pytest.mark.parametrize("graph,cin,B,T", [("h1389", 2, 3, 12), ("pems_bay", 4, 5, 3), ("h2600", 1, 2, 1), ("smallest", 2, 4, 2)])
def test_fused_training_vs_autograd(graph, cin, B, T):
    n, ei, ew = _graph_case(graph)
    X = torch.randn(B, T, n, cin, device=DEV)
    w = torch.randn(B, T, n, 32, device=DEV)
    for bias in (True, False):
        m = _model(cin, 7, bias)
        for x_grad in (True, False):
            res = []
            for fused in (True, False):
                m._fused_training = fused
                with _counted() as c:
                    res.append(_train(m, X, ei, ew, w, x_grad))
                assert (c.get("k_dcrnn_rows_bwd_start", 0) == 1) == fused and (c.get("k_spmm", 0) > 0) != fused
                assert c.get("k_dcrnn_rows_bwd_x", 0) == int(fused and x_grad)
            m._fused_training = True
            (of, *gf), (oa, *ga) = res
            _close(of, oa)
            for a, b in zip(gf, ga):
                assert (a is None) == (b is None)
                if b is not None:
                    _grad_close(a, b)


def test_training_forward_is_bit_equal_and_backward_deterministic_and_scale_equivariant():
    n, ei, ew = _graph_case("h1389")
    m = _model(2, 3)
    X = torch.randn(3, 12, n, 2, device=DEV)
    w = torch.randn(3, 12, n, 32, device=DEV)
    with torch.no_grad():
        ref = m(X, ei, ew)
    base = _train(m, X, ei, ew, w)
    assert torch.equal(base[0], ref)
    again = _train(m, X, ei, ew, w)
    assert all(torch.equal(a, b) for a, b in zip(again, base))
    for e in (-24, 8):
        scaled = _train(m, X, ei, ew, w * 2.0 ** e)
        assert all(torch.equal(a, b * 2.0 ** e) for a, b in zip(scaled[1:], base[1:]))


def test_forward_indexed_equals_materialised_windows_and_empty_calls():
    ei, ew, series = synthetic.pems_bay_like(0, 300)
    ei, ew, s = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV), torch.from_numpy(series).to(DEV)
    m = _model(2, 1)
    starts = torch.randint(0, 300 - 12, (64,), generator=torch.Generator().manual_seed(0)).to(DEV)
    X = torch.stack([s[i:i + 12] for i in starts.tolist()])
    with torch.no_grad():
        with _counted() as c:
            a = m.forward_indexed(s, starts, 12, ei, ew)
        assert "k_window_gather" not in c and c["k_dcrnn_rows_fwd_a"] == 12
        assert torch.equal(a, m(X, ei, ew))
        e0 = m.forward_indexed(s, starts[:0], 12, ei, ew)
        e1 = m(X[:, :0], ei, ew)
    assert e0.shape == (0, 12, 325, 32) and e1.shape == (64, 0, 325, 32)
    for Xe in (X[:0], X[:, :0]):
        out = m(Xe.clone().requires_grad_(True), ei, ew)
        out.sum().backward()
        assert out.shape == Xe.shape[:3] + (32,)
        assert all(bool((p.grad == 0).all()) for p in m.parameters())
        m.zero_grad(set_to_none=True)


# ---- a PeMS-like size: the weight-gradient bases pass 2^31 bytes ----------------------------------------------------------------------
def test_pems_like_size_training_step_vs_tiled():
    n, B, T = 11160, 64, 12
    ei, ew = _graph(n, 8, 11)
    m = _model(2, 5)
    X = torch.randn(B, T, n, 2, device=DEV)
    w = torch.randn(B, T, n, 32, device=DEV)
    ld = ops.dcrnn_bwd_basis_ld(2, 32, 2)
    assert T * B * n * ld * 4 > 2 ** 31
    res = []
    for fused in (True, False):
        m._fused_training = fused
        res.append(_train(m, X, ei, ew, w, x_grad=False))
        torch.cuda.empty_cache()
    m._fused_training = True
    (of, *gf), (oa, *ga) = res
    _close(of, oa)
    for a, b in zip(gf[1:], ga[1:]):
        _grad_close(a, b)


# ---- a captured training step -----------------------------------------------------------------------------------------------------------
def test_cuda_graph_training_step_equals_eager():
    """forward, masked MAE, backward and FlatAdam captured once and replayed equal the same steps run eagerly."""
    ei, ew, series = synthetic.pems_bay_like(0, 200)
    ei, ew, s = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV), torch.from_numpy(series).to(DEV)
    batches = [(s[i:i + 12].unsqueeze(0).repeat(4, 1, 1, 1), s[i + 12:i + 24, :, :1].unsqueeze(0).repeat(4, 1, 1, 32)) for i in (0, 30, 60, 90)]

    def make():
        m = _model(2, 9)
        sync = D.FlatGradSync(m.parameters())
        return m, D.FlatAdam(sync, lr=1e-3)

    m, opt = make()
    xs, ys = batches[0][0].clone(), batches[0][1].clone()

    def step():
        loss = ops.masked_mae(m(xs, ei, ew), ys)
        loss.backward()
        opt.step()
        return loss

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step()
    m_e, opt_e = make()
    for _ in range(2):                                     # bring the eager twin to the state the capture started from
        ops.masked_mae(m_e(batches[0][0], ei, ew), batches[0][1]).backward()
        opt_e.step()
    for p, pe in zip(m.parameters(), m_e.parameters()):
        assert torch.equal(p, pe)
    for x, y in batches:
        xs.copy_(x)
        ys.copy_(y)
        graph.replay()
        le = ops.masked_mae(m_e(x, ei, ew), y)
        le.backward()
        opt_e.step()
        assert torch.equal(loss, le.detach())
    torch.cuda.synchronize()
    for p, pe in zip(m.parameters(), m_e.parameters()):
        assert torch.equal(p, pe)


# ---- routing, launch budget, ABI ------------------------------------------------------------------------------------------------------
def test_routing():
    """Graphs that fit one SM keep the one-SM kernels; cout 16, K = 3, cin 5 and the DCRNN cell at 325 nodes stay on the tiled path."""
    e, w, _ = synthetic.metr_la_like(0, 16)
    ei, ew = torch.from_numpy(e).to(DEV), torch.from_numpy(w).to(DEV)
    m = _model(2, 0)
    X = torch.randn(2, 3, 207, 2, device=DEV)
    with _counted() as c, torch.no_grad():
        m(X, ei, ew)
    assert "k_dcrnn_seq_tc" in c and not any(k in c for k in ROWS)
    with _counted() as c:
        m(X, ei, ew).sum().backward()
    assert not any(k in c for k in ROWS)
    _lib.set_option("dcrnn_tc", 0)
    try:
        with _counted() as c, torch.no_grad():
            m(X, ei, ew)
        assert "k_dcrnn_seq" in c and not any(k in c for k in ROWS)
    finally:
        _lib.set_option("dcrnn_tc", 1)
    e, w, _ = synthetic.pems_bay_like(0, 16)
    ei, ew = torch.from_numpy(e).to(DEV), torch.from_numpy(w).to(DEV)
    for cin, cout, K in ((2, 16, 2), (2, 32, 3), (5, 32, 2)):
        mm = BatchedDCRNN(cin, cout, K).to(DEV)
        X = torch.randn(2, 3, 325, cin, device=DEV)
        with _counted() as c:
            with torch.no_grad():
                mm(X, ei, ew)
            mm(X, ei, ew).sum().backward()
        assert "k_spmm" in c and not any(k in c for k in ROWS), (cin, cout, K)
    cell = DCRNN(2, 32, 2).to(DEV)
    with _counted() as c:
        cell(torch.randn(325, 2, device=DEV), ei, ew).sum().backward()
    assert "k_spmm" in c and not any(k in c for k in ROWS)


def test_training_step_launch_budget():
    ei, ew, series = synthetic.pems_bay_like(0, 64)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    X = torch.from_numpy(series[:48]).reshape(4, 12, 325, 2).to(DEV).repeat(16, 1, 1, 1)        # B = 64, T = 12
    m = _model(2, 0)
    w = torch.ones(64, 12, 325, 32, device=DEV)
    _train(m, X, ei, ew, w, x_grad=False)                   # plan, packed weights and workspaces warm
    n0 = _lib.launch_count()
    out = m(X, ei, ew)
    assert _lib.launch_count() - n0 == 2 * 12 - 1
    (out * w).sum().backward()
    assert _lib.launch_count() - n0 == (2 * 12 - 1) + (2 * 12 - 1) + 2      # forward, backward, wgrad contraction + reduce


def test_abi_errors():
    ei, ew, _ = synthetic.pems_bay_like(0, 16)
    dconv = GraphPlan(_lib.FLAVOR_DCONV, torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV), 325, flags=_lib.DCONV_ALLOW_DUPLICATES)
    cheb = GraphPlan(_lib.FLAVOR_CHEB, torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV), 325, "sym")
    L = _lib.lib()
    h = dconv.handle
    buf = torch.zeros(1 << 22, device=DEV)
    p, q = _lib.ptr(buf), ctypes.c_void_p(buf.data_ptr() + 4)       # q: 4-byte aligned only
    r = ctypes.c_void_p(buf.data_ptr() + 2)                         # r: misaligned
    assert L.stmp_dcrnn_rows_supported(h, 4, 32, 2) == 1 and L.stmp_dcrnn_rows_supported(h, 1, 32, 2) == 1
    assert L.stmp_dcrnn_rows_supported(h, 5, 32, 2) == 0 and L.stmp_dcrnn_rows_supported(h, 2, 16, 2) == 0
    assert L.stmp_dcrnn_rows_supported(h, 2, 32, 3) == 0 and L.stmp_dcrnn_rows_supported(None, 2, 32, 2) == 0
    assert L.stmp_dcrnn_rows_supported(cheb.handle, 2, 32, 2) == 0
    assert L.stmp_dcrnn_rows_scratch_bytes(h, 3) == 3 * 325 * 256 * 4 and L.stmp_dcrnn_rows_scratch_bytes(None, 3) == 0
    ld = ops.dcrnn_bwd_basis_ld(2, 32, 2)

    def fwd(plan=h, B=1, cin=2, x=p, w=p, S1=p, S2=p, st=p, ldv=ld):
        return L.stmp_dcrnn_rows_fwd(plan, B, 1, cin, x, None, 0, 0, w, p, None, None, None, p, p, st, S1, S2, ldv, None)
    assert fwd(plan=None) == _lib.STMP_EINVAL and fwd(plan=cheb.handle) == _lib.STMP_EINVAL and fwd(B=-1) == _lib.STMP_EINVAL
    assert fwd(cin=5) == _lib.STMP_EUNSUPPORTED and fwd(cin=0) == _lib.STMP_EUNSUPPORTED
    assert fwd(x=None) == _lib.STMP_EINVAL and fwd(w=None) == _lib.STMP_EINVAL and fwd(S2=None) == _lib.STMP_EINVAL
    assert fwd(ldv=ld + 8) == _lib.STMP_ESHAPE and fwd(x=r) == _lib.STMP_ESHAPE and fwd(S1=q) == _lib.STMP_ESHAPE
    assert fwd(B=1 << 23) == _lib.STMP_ESHAPE
    assert fwd(B=0) == _lib.STMP_OK

    def bwd(plan=h, cin=2, g=p, st=p, dx=None):
        return L.stmp_dcrnn_rows_bwd(plan, 1, 1, cin, g, p, st, p, p, p, p, p, dx, None)
    assert bwd(plan=None) == _lib.STMP_EINVAL and bwd(plan=cheb.handle) == _lib.STMP_EINVAL and bwd(cin=5) == _lib.STMP_EUNSUPPORTED
    assert bwd(g=None) == _lib.STMP_EINVAL and bwd(st=None) == _lib.STMP_EINVAL and bwd(g=r) == _lib.STMP_ESHAPE
    assert bwd(dx=r) == _lib.STMP_ESHAPE
