"""BatchedDCRNN at 64 hidden channels (the DCRNN paper's width), K = 2 and 3, on any graph: the 64-wide row-split kernels
(`stmp_dcrnn_wide_rows_*`, DESIGN §4m).  BatchedDCRNN(2, 64, 3) on the METR-LA shape and (2, 64, 2) on the PEMS-BAY shape against the
unmodified reference (tests/golden/make_goldens_dcrnn_wide_rows.py); the forward against the float64 oracle across cin x K on METR-LA,
PEMS-BAY, 1000-2600-node graphs with 400-edge hubs and isolated nodes and 50 000 nodes, with B in {1, 3, 64} and T in {1, 2, 12}; the
reference's non-finite pattern; fused training against autograd through the tiled path; bit-identity, determinism and loss-scale
equivariance; index batching and empty calls; an 11 160-node training step; a captured training step; routing, the launch budget and the
C ABI's errors."""
import contextlib
import ctypes
import gzip
import importlib.util
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
WROWS = ("k_dcrnn_wrows_image", "k_dcrnn_wrows_fwd0", "k_dcrnn_wrows_fwd", "k_dcrnn_wrows_bwd0", "k_dcrnn_wrows_bwd")


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
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _grad_close(got, ref):
    _close(got, ref, 1e-3, 1e-3 * max(ref.abs().max().item(), 1e-12))


def _golden_module():
    spec = importlib.util.spec_from_file_location("_mk_wrows", os.path.join(os.path.dirname(__file__), "golden",
                                                                            "make_goldens_dcrnn_wide_rows.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _graph(n, deg, seed, hubs=False):
    """Random directed graph plus a ring (every DConv norm finite); with `hubs`, node 0 gets 400 in-edges and node 1 400 out-edges, and
    nodes 2..11 have no edge at all: isolated, so they hold no operator entry and their rows see only X."""
    g = torch.Generator().manual_seed(seed)
    src, dst = torch.randint(0, n, (deg * n,), generator=g), torch.randint(0, n, (deg * n,), generator=g)
    r = torch.arange(n)
    if hubs:
        keep = (src >= 12) & (dst >= 12)
        src, dst = src[keep], dst[keep]
        pick = torch.randperm(n - 12, generator=g)[:400] + 12
        src, dst = torch.cat([src, pick, torch.ones(400, dtype=torch.long)]), torch.cat([dst, torch.zeros(400, dtype=torch.long), pick])
        ring = torch.cat([torch.tensor([0, 1]), torch.arange(12, n)])
        src, dst = torch.cat([src, ring]), torch.cat([dst, ring.roll(-1)])
    else:
        src, dst = torch.cat([src, r]), torch.cat([dst, (r + 1) % n])
    ei = torch.unique(torch.stack([src, dst]), dim=1)
    ei = ei[:, ei[0] != ei[1]]
    return ei.to(DEV), (torch.rand(ei.size(1), generator=g) + 0.1).to(DEV)


def _banded(n, seed):
    ei, ew = synthetic.banded_graph(n, 8 * n, span=32, seed=seed)
    r = torch.arange(n)
    ei = torch.cat([torch.from_numpy(ei), torch.stack([r, (r + 1) % n])], 1)
    ew = torch.cat([torch.from_numpy(ew), torch.full((n,), 0.5)])
    return ei.to(DEV), ew.to(DEV)


def _like(name):
    like, n = {"metr_la": (synthetic.metr_la_like, 207), "pems_bay": (synthetic.pems_bay_like, 325)}[name]
    e, w, _ = like(0, 16)
    return n, torch.from_numpy(e).to(DEV), torch.from_numpy(w).to(DEV)


def _graph_case(name):
    if name in ("metr_la", "pems_bay"):
        return _like(name)
    if name == "hub1000":
        return (1000,) + _graph(1000, 6, 10, hubs=True)
    if name == "hub2600":
        return (2600,) + _graph(2600, 8, 26, hubs=True)
    if name == "banded2000":
        return (2000,) + _banded(2000, 3)
    if name == "n11160":
        return (11160,) + _banded(11160, 11)
    if name == "n50000":
        return (50000,) + _graph(50000, 4, 50)
    raise KeyError(name)


def _plan(ei, ew, n):
    return GraphPlan(_lib.FLAVOR_DCONV, ei, ew, n, flags=_lib.DCONV_ALLOW_DUPLICATES)


def _model(cin, K, seed, bias=True):
    torch.manual_seed(seed)
    m = BatchedDCRNN(cin, 64, K, bias=bias)
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


def _fwd_launches(K, T, nonfinite=False):
    """the forward launch budget of DESIGN §4m: the weight image, then 2(K-1) per step and one for step 0"""
    return 1 + (2 * (K - 1) * T if nonfinite else 1 + 2 * (K - 1) * (T - 1))


def _bwd_launches(K, T):
    return 2 + 2 * (K - 1) * (T - 1)


def _chunks(n, cin, K, B, T):
    """window chunks of a no_grad call: the hoisted X blocks of one chunk stay under ops._NROWS_XBUF_BYTES"""
    per = max(1, min(B, ops._NROWS_XBUF_BYTES // (T * n * (2 * K - 1) * cin * 4)))
    return -(-B // per)


def _wrows(c):
    return sum(v for k, v in c.items() if k in WROWS)


# ---- the goldens from the unmodified reference ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["metr_la", "pems_bay"])
def test_golden(golden_dir, name):
    """The golden holds the reference's float64 values.  The output is held to rtol 1e-4 with atol 2e-5: on METR-LA at K = 3 one element
    of the exact-fp32 result measured 1.5e-5 from the exact value (a float32 run of the reference lands about as far), while the
    forward's float64-oracle test bounds the error by 8x the float32 oracle's everywhere."""
    mk = _golden_module()
    with gzip.open(os.path.join(golden_dir, f"dcrnn_wide_rows_{name}.pt.gz"), "rb") as f:
        g = torch.load(f, weights_only=False)
    steps = g["out_steps"]
    ei, ew, X, K = mk.inputs(name)
    ei, ew, X = ei.to(DEV), ew.to(DEV), X.to(DEV)
    m = BatchedDCRNN(2, 64, K).to(DEV)
    m.load_state_dict({k: v for k, v in mk.params([(n_, p.shape) for n_, p in m.named_parameters()], 11).items()})
    T, N = X.size(1), X.size(2)
    with _counted() as c, torch.no_grad():
        out = m(X, ei, ew)
    assert _wrows(c) == _fwd_launches(K, T) and c["k_spmm"] == 2 * (K - 1)
    _close(out[:, steps], g["out"], atol=2e-5)
    Xl = X.clone().requires_grad_(True)
    with _counted() as c:
        out = m(Xl, ei, ew)
        (out * torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)).sum().backward()
    assert c["k_dcrnn_wrows_bwd"] == 2 * (K - 1) * (T - 1) and c["k_spmm"] == 4 * (K - 1)
    _close(out[:, steps], g["out"], atol=2e-5)
    _grad_close(Xl.grad, g["gX"])
    for k, p in m.named_parameters():
        _grad_close(p.grad, g["grads"][k])


# ---- against the float64 oracle -------------------------------------------------------------------------------------------------------
# (graph, cin, K, B, T): every cin and K, B in {1, 3, 64}, T in {1, 2, 12}
CASES = [("metr_la", 2, 3, 64, 12), ("metr_la", 1, 2, 3, 1), ("pems_bay", 2, 2, 64, 12), ("pems_bay", 4, 3, 1, 2),
         ("hub1000", 3, 3, 3, 12), ("hub1000", 1, 2, 64, 2), ("hub2600", 4, 2, 3, 12), ("hub2600", 2, 3, 1, 1),
         ("n50000", 2, 3, 3, 12), ("n50000", 3, 2, 1, 2)]


@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_forward_vs_float64_oracle(case):
    """Criterion: at most 8x the error of the same oracle in float32, plus 2^-20 of the output's scale (a 400-entry hub row sums in CSR
    order, where the float32 oracle's scatter order can land closer by chance)."""
    graph, cin, K, B, T = case
    n, ei, ew = _graph_case(graph)
    m = _model(cin, K, cin + T)
    X = torch.randn(B, T, n, cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(B + T))
    plan = m._plan(ei, ew, n)
    assert not ops.dcrnn_seq_supported(plan, cin, 64, K) and ops.dcrnn_wide_rows_supported(plan, cin, 64, K)
    with _counted() as c, torch.no_grad():
        out = m(X, ei, ew)
    ch = _chunks(n, cin, K, B, T)
    assert _wrows(c) == ch * _fwd_launches(K, T) and c.get("k_spmm", 0) == ch * 2 * (K - 1)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    with torch.no_grad():
        ref32 = R.batched_dcrnn(sd, X, ei, ew)
        with _float64():
            ref64 = R.batched_dcrnn({k: v.double() for k, v in sd.items()}, X.double(), ei, ew.double())
    got = out.double()
    assert bool(torch.isfinite(got).all())
    e32 = float((ref32.double() - ref64).abs().max())
    e, scale = float((got - ref64).abs().max()), float(ref64.abs().max())
    assert e <= 8 * e32 + 2.0 ** -20 * scale, (case, e, e32, scale)


def test_zero_degree_nodes_give_the_reference_non_finite_pattern():
    """A path graph of 1500 nodes: node 0 has no in-edge, so DConv's 1/deg_in is inf on its out-edge.  inf * 0 = NaN reaches the state at
    step 0 and spreads from there -- the reference's pattern, which needs the full chain at step 0."""
    n = 1500
    ei = torch.stack([torch.arange(n - 1), torch.arange(1, n)]).to(DEV)
    ew = torch.ones(n - 1, device=DEV)
    for K in (2, 3):
        m = _model(2, K, 0)
        X = torch.randn(2, 4, n, 2, device=DEV)
        want = R.batched_dcrnn({k: v.detach() for k, v in m.state_dict().items()}, X, ei, ew)
        assert not bool(torch.isfinite(want).all()) and bool(torch.isfinite(want).any())
        for grad in (False, True):
            with _counted() as c, torch.set_grad_enabled(grad):
                got = m(X, ei, ew).detach()
            assert c.get("k_dcrnn_wrows_fwd") == 2 * (K - 1) * 4 and "k_dcrnn_wrows_fwd0" not in c
            assert torch.equal(torch.isfinite(got), torch.isfinite(want))
            fin = torch.isfinite(want)
            _close(got[fin], want[fin])


# ---- training: fused against autograd through the tiled path ---------------------------------------------------------------------------
@pytest.mark.parametrize("graph,cin,K,B,T", [("metr_la", 2, 3, 3, 12), ("pems_bay", 4, 2, 5, 3), ("banded2000", 1, 3, 2, 1),
                                             ("banded2000", 3, 2, 33, 2)])
def test_fused_training_vs_autograd(graph, cin, K, B, T):
    n, ei, ew = _graph_case(graph)
    X = torch.randn(B, T, n, cin, device=DEV)
    w = torch.randn(B, T, n, 64, device=DEV)
    for bias in (True, False):
        m = _model(cin, K, 7, bias)
        for x_grad in (True, False):
            res = []
            for fused in (True, False):
                m._fused_training = fused
                with _counted() as c:
                    res.append(_train(m, X, ei, ew, w, x_grad))
                assert (_wrows(c) == _fwd_launches(K, T) + _bwd_launches(K, T)) == fused and (_wrows(c) == 0) != fused
            m._fused_training = True
            (of, *gf), (oa, *ga) = res
            _close(of, oa)
            for a, b in zip(gf, ga):
                assert (a is None) == (b is None)
                if b is not None:
                    _grad_close(a, b)


@pytest.mark.parametrize("K", [2, 3])
def test_training_forward_is_bit_equal_and_backward_deterministic_and_scale_equivariant(K):
    n, ei, ew = _graph_case("banded2000")
    m = _model(2, K, 3)
    X = torch.randn(3, 12, n, 2, device=DEV)
    w = torch.randn(3, 12, n, 64, device=DEV)
    with torch.no_grad():
        ref = m(X, ei, ew)
    base = _train(m, X, ei, ew, w)
    assert torch.equal(base[0], ref)
    again = _train(m, X, ei, ew, w)
    assert all(torch.equal(a, b) for a, b in zip(again, base))
    for e in (-24, 8):
        scaled = _train(m, X, ei, ew, w * 2.0 ** e)
        assert all(torch.equal(a, b * 2.0 ** e) for a, b in zip(scaled[1:], base[1:]))


@pytest.mark.parametrize("K", [2, 3])
def test_forward_indexed_equals_materialised_windows_and_empty_calls(K):
    n, ei, ew = _like("metr_la")
    s = torch.randn(300, n, 2, device=DEV)
    m = _model(2, K, 1)
    starts = torch.randint(0, 300 - 12, (64,), generator=torch.Generator().manual_seed(0)).to(DEV)
    X = torch.stack([s[i:i + 12] for i in starts.tolist()])
    with torch.no_grad():
        with _counted() as c:
            a = m.forward_indexed(s, starts, 12, ei, ew)
        assert c["k_dcrnn_wrows_fwd"] == 2 * (K - 1) * 11 and c["k_window_gather"] == 1
        assert torch.equal(a, m(X, ei, ew))
        e0 = m(X[:0], ei, ew)
        e1 = m(X[:, :0], ei, ew)
    assert e0.shape == (0, 12, n, 64) and e1.shape == (64, 0, n, 64)
    for Xe in (X[:0], X[:, :0]):
        out = m(Xe.clone().requires_grad_(True), ei, ew)
        out.sum().backward()
        assert out.shape == Xe.shape[:3] + (64,)
        assert all(bool((p.grad == 0).all()) for p in m.parameters())
        m.zero_grad(set_to_none=True)


# ---- a large graph ----------------------------------------------------------------------------------------------------------------------
def test_11160_node_training_step_vs_tiled():
    """BatchedDCRNN(2, 64, 3) at 11 160 nodes, B = 16 windows of 12 steps: the tiled path's autograd graph at B = 64 would not fit 80 GB
    next to the fused path's bases (each about 11 GB at B = 64), so both run at B = 16."""
    n, B, T = 11160, 16, 12
    ei, ew = _banded(n, 11)
    m = _model(2, 3, 5)
    X = torch.randn(B, T, n, 2, device=DEV)
    w = torch.randn(B, T, n, 64, device=DEV)
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
    n, ei, ew = _like("metr_la")
    s = torch.randn(200, n, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    batches = [(s[i:i + 12].unsqueeze(0).repeat(4, 1, 1, 1), s[i + 12:i + 24, :, :1].expand(12, n, 64).unsqueeze(0).repeat(4, 1, 1, 1))
               for i in (0, 30, 60, 90)]

    def make():
        m = _model(2, 3, 9)
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
    for _ in range(2):
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
    """(2, 64, 2) and (2, 64, 3) take the new kernels on METR-LA and on large graphs; 32-wide and narrow models keep their kernels;
    `_fused_training = False` keeps the tiled path for training; cout 64 at K 1 or 4, cin 5 and the DCRNN cell stay off the new kernels."""
    n, ei, ew = _like("metr_la")
    for K in (2, 3):
        m = _model(2, K, 0)
        X = torch.randn(2, 3, n, 2, device=DEV)
        with _counted() as c, torch.no_grad():
            m(X, ei, ew)
        assert c.get("k_dcrnn_wrows_fwd0") == 1
        with _counted() as c:
            m(X, ei, ew).sum().backward()
        assert "k_dcrnn_wrows_bwd" in c
        m._fused_training = False
        with _counted() as c:
            m(X, ei, ew).sum().backward()
        assert "k_spmm" in c and _wrows(c) == 0
    n, ei, ew = _graph_case("banded2000")
    for cout, K, kern in ((32, 2, "k_dcrnn_rows_fwd_a"), (2, 3, "k_dcrnn_nrows_fwd")):
        m = BatchedDCRNN(2, cout, K).to(DEV)
        with _counted() as c, torch.no_grad():
            m(torch.randn(2, 3, n, 2, device=DEV), ei, ew)
        assert kern in c and _wrows(c) == 0
    for cin, K in ((2, 1), (2, 4), (5, 2)):
        mm = BatchedDCRNN(cin, 64, K).to(DEV)
        with _counted() as c, torch.no_grad():
            mm(torch.randn(2, 3, n, cin, device=DEV), ei, ew)
        assert _wrows(c) == 0 and ("k_spmm" in c) == (K > 1), (cin, K)
    n, ei, ew = _graph_case("hub1000")                          # no duplicate edges: the DCRNN cell's DConv refuses them
    cell = DCRNN(2, 64, 3).to(DEV)
    with _counted() as c:
        cell(torch.randn(n, 2, device=DEV), ei, ew).sum().backward()
    assert _wrows(c) == 0


@pytest.mark.parametrize("K", [2, 3])
def test_training_step_launch_budget(K):
    """DESIGN §4m: forward = the weight image + 2(K-1) launches per step, one for step 0, plus 2(K-1) hoisted SpMMs over X; backward =
    the weight image + 1 + 2(K-1)(T-1) launches, plus the weight-gradient products; no other library launch."""
    n, ei, ew = _like("pems_bay")
    m = _model(2, K, 0)
    X = torch.randn(64, 12, n, 2, device=DEV)
    w = torch.ones(64, 12, n, 64, device=DEV)
    _train(m, X, ei, ew, w, x_grad=False)                   # plan and packed weights warm
    n0 = _lib.launch_count()
    out = m(X, ei, ew)
    assert _lib.launch_count() - n0 == _fwd_launches(K, 12) + 2 * (K - 1)
    (out * w).sum().backward()
    assert _lib.launch_count() - n0 == _fwd_launches(K, 12) + 2 * (K - 1) + _bwd_launches(K, 12)


def test_abi_errors():
    n, ei, ew = _graph_case("banded2000")
    dconv = _plan(ei, ew, n)
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei, ew, n, "sym")
    L = _lib.lib()
    h = dconv.handle
    buf = torch.zeros(1 << 22, device=DEV)
    p, q = _lib.ptr(buf), ctypes.c_void_p(buf.data_ptr() + 4)       # q: 4-byte aligned only
    r = ctypes.c_void_p(buf.data_ptr() + 2)                         # r: misaligned
    S = L.stmp_dcrnn_wide_rows_supported
    assert S(h, 4, 64, 3) == 1 and S(h, 1, 64, 2) == 1 and S(h, 5, 64, 3) == 0 and S(h, 2, 32, 2) == 0 and S(h, 2, 64, 4) == 0
    assert S(h, 2, 64, 1) == 0 and S(h, 0, 64, 3) == 0 and S(None, 2, 64, 3) == 0 and S(cheb.handle, 2, 64, 3) == 0
    img = 2 * 340 * 192 * 4
    assert L.stmp_dcrnn_wide_rows_scratch_bytes(h, 3, 64, 3) == img + 10 * n * 3 * 64 * 4
    assert L.stmp_dcrnn_wide_rows_scratch_bytes(h, 3, 64, 1) == 0 and L.stmp_dcrnn_wide_rows_scratch_bytes(None, 3, 64, 3) == 0
    assert L.stmp_dcrnn_wide_rows_scratch_bytes(h, 3, 32, 2) == 0

    def fwd(plan=h, B=1, T=1, cin=2, cout=64, K=3, x=p, w=p, scr=p, out=p, S1=None, S2=None, st=None, xld=10):
        return L.stmp_dcrnn_wide_rows_fwd(plan, B, T, cin, cout, K, x, 0, 0, xld, 2, w, p, None, None, None, scr, out, st, S1, S2, None)
    assert fwd(plan=None) == _lib.STMP_EINVAL and fwd(plan=cheb.handle) == _lib.STMP_EINVAL and fwd(B=-1) == _lib.STMP_EINVAL
    assert fwd(cin=5) == _lib.STMP_EUNSUPPORTED and fwd(cout=32) == _lib.STMP_EUNSUPPORTED and fwd(K=4) == _lib.STMP_EUNSUPPORTED
    assert fwd(x=None) == _lib.STMP_EINVAL and fwd(w=None) == _lib.STMP_EINVAL and fwd(scr=None) == _lib.STMP_EINVAL
    assert fwd(S1=p) == _lib.STMP_EINVAL and fwd(S1=p, S2=p) == _lib.STMP_EINVAL
    assert fwd(x=r) == _lib.STMP_ESHAPE and fwd(scr=q) == _lib.STMP_ESHAPE and fwd(out=q) == _lib.STMP_ESHAPE
    assert fwd(xld=1) == _lib.STMP_ESHAPE
    assert fwd(B=(1 << 40) // n + 1) == _lib.STMP_ESHAPE and fwd(T=1 << 31) == _lib.STMP_ESHAPE   # refused before any launch
    assert fwd(B=0) == _lib.STMP_OK and fwd(T=0) == _lib.STMP_OK

    def bwd(plan=h, cin=2, K=3, g=p, st=p, dsx=None, ld=10):
        return L.stmp_dcrnn_wide_rows_bwd(plan, 1, 1, cin, 64, K, g, p, st, p, p, p, p, p, dsx, ld, None)
    assert bwd(plan=None) == _lib.STMP_EINVAL and bwd(plan=cheb.handle) == _lib.STMP_EINVAL and bwd(cin=5) == _lib.STMP_EUNSUPPORTED
    assert bwd(K=1) == _lib.STMP_EUNSUPPORTED and bwd(g=None) == _lib.STMP_EINVAL and bwd(st=None) == _lib.STMP_EINVAL
    assert bwd(g=q) == _lib.STMP_ESHAPE and bwd(st=q) == _lib.STMP_ESHAPE and bwd(dsx=r) == _lib.STMP_ESHAPE
    assert bwd(dsx=p, ld=9) == _lib.STMP_ESHAPE
