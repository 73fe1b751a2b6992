"""GConvGRU on graphs larger than one SM: the row-split cell kernels (`stmp_gru_rows_*`, DESIGN §4i).  The reference's WikiMaths tutorial
against the unmodified reference (tests/golden/make_goldens_wikimaths.py), fused and op-for-op; launch counts; bit-equality of training
and inference forwards; determinism and loss-scale equivariance of the backward; the row-split kernels against the one-SM kernel at the
ops level; the fused path against op-for-op autograd on random graphs with hubs and isolated nodes; a captured tutorial step; routing;
and the C ABI's errors."""
import ctypes

import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU
from pytorch_geometric_temporal_b200.plan import GraphPlan
from gconvgru_seq import chickenpox_train_split
from wikimaths_seq import load, model_for, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = ["K2_sym", "K1_sym", "K2_sym_carried", "K2_rw"]
ROWS = ("k_gru_rows_fwd_a", "k_gru_rows_fwd_b", "k_gru_rows_bwd_a", "k_gru_rows_bwd_b", "k_gru_rows_bwd_c", "k_dcrnn_wgrad",
        "k_gru_rows_wgrad_reduce")


def _ran(before, name):
    return _lib.path_counters().get(name, 0) - before.get(name, 0)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _close_grad(got, want):
    _close(got, want, 1e-3, 1e-3 * want.abs().max().item() + 1e-6)


def _structurally_zero(name):
    """Parameters whose gradient is exactly zero with H = None: every conv_h_* weight, conv_x_r and both r biases."""
    return (name.startswith("recurrent.conv_h_") and ".lins." in name) or name.startswith("recurrent.conv_x_r.") or name == "recurrent.conv_h_r.bias"


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", CASES)
def test_wikimaths_vs_reference_golden(golden_dir, case, fused):
    g = load(golden_dir)
    c = g["cases"][case]
    m = model_for(c, DEV, fused)
    H0 = c["H0"].to(DEV).requires_grad_(True) if "H0" in c else None
    c0 = _lib.path_counters()
    out, losses = run(m, g, c, DEV, H0)
    S = g["X"].shape[0]
    if fused:
        assert _ran(c0, "k_gru_rows_fwd_a") == S and _ran(c0, "k_gru_rows_bwd_a") == S and _ran(c0, "k_spmm") == 0
        assert _ran(c0, "k_gru_rows_fwd_b") == (S if H0 is not None else 0)
    else:
        assert all(_ran(c0, k) == 0 for k in ROWS)
    _close(out, c["out"])
    _close(losses, c["losses"])
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        _close_grad(p.grad, c["grads"][k])
        if H0 is None and _structurally_zero(k):
            assert torch.all(p.grad == 0), k
    if H0 is not None:
        _close_grad(H0.grad, c["gH0"])


def _wiki_graph(golden_dir):
    g = load(golden_dir)
    return g["edge_index"].to(DEV).long(), g["edge_weight"].to(DEV), g["X"].to(DEV)


def _cell(cin, K, N, norm="sym", bias=True, seed=0):
    torch.manual_seed(seed)
    m = GConvGRU(cin, 32, K, normalization=norm, bias=bias).to(DEV)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn_like(p) * 0.1)
    return m, torch.randn(N, cin, device=DEV), torch.randn(N, 32, device=DEV) * 0.5, torch.randn(N, 32, device=DEV)


def test_launch_counts(golden_dir):
    ei, ew, X = _wiki_graph(golden_dir)
    m, _, H, w = _cell(14, 2, X.size(1))
    x = X[0]
    Hl = H.clone().requires_grad_(True)
    (m(x, ei, ew, Hl) * w).sum().backward()                    # warm: plan, packed weights, workspaces
    for h, want in ((H, 2), (None, 1)):
        n0 = _lib.launch_count()
        with torch.no_grad():
            m(x, ei, ew, h)
        assert _lib.launch_count() - n0 == want
    n0 = _lib.launch_count()
    (m(x, ei, ew) * w).sum().backward()                        # the tutorial: H = None, X needs no gradient
    assert _lib.launch_count() - n0 == 4                       # fwd_a, bwd_a, wgrad contraction, reduce
    xl = x.clone().requires_grad_(True)
    c0, n0 = _lib.path_counters(), _lib.launch_count()
    (m(xl, ei, ew, Hl) * w).sum().backward()
    assert _lib.launch_count() - n0 == 7
    assert {k: _ran(c0, k) for k in ROWS + ("k_spmm",)} == {**{k: 1 for k in ROWS}, "k_spmm": 0}


def test_training_forward_is_bit_equal_to_inference_and_backward_is_deterministic(golden_dir):
    ei, ew, X = _wiki_graph(golden_dir)
    for K in (1, 2):
        m, _, H, w = _cell(14, K, X.size(1), seed=K)
        x = X[1]
        for h in (H, None):
            out = m(x, ei, ew, h)
            assert out.requires_grad
            with torch.no_grad():
                assert torch.equal(out.detach(), m(x, ei, ew, h))

            def grads():
                m.zero_grad(set_to_none=True)
                xl = x.clone().requires_grad_(True)
                hl = None if h is None else h.clone().requires_grad_(True)
                (m(xl, ei, ew, hl) * w).sum().backward()
                return [xl.grad] + ([hl.grad] if hl is not None else []) + [p.grad.clone() for p in m.parameters()]
            for a, b in zip(grads(), grads()):
                assert torch.equal(a, b)


@pytest.mark.parametrize("case", ["K2_sym", "K2_sym_carried"])
def test_gradients_scale_with_a_power_of_two_loss_scale_bit_for_bit(golden_dir, case):
    g = load(golden_dir)
    c = g["cases"][case]

    def grads(scale):
        m = model_for(c, DEV, True)
        H0 = c["H0"].to(DEV).requires_grad_(True) if "H0" in c else None
        c0 = _lib.path_counters()
        ei, ew, X, Y = g["edge_index"].to(DEV).long(), g["edge_weight"].to(DEV), g["X"].to(DEV), g["Y"].to(DEV)
        h, total = H0, 0
        for t in range(X.shape[0]):
            hh = m.recurrent(X[t], ei, ew) if H0 is None else m.recurrent(X[t], ei, ew, h)
            h = hh
            total = total + torch.mean((m.linear(torch.relu(hh)).squeeze() - Y[t]) ** 2)
        (total * scale).backward()
        assert _ran(c0, "k_gru_rows_bwd_a") == X.shape[0]
        return [p.grad for p in m.parameters()] + ([H0.grad] if H0 is not None else [])
    base = grads(1.0)
    for e in (-24, 8):
        for a, b in zip(grads(2.0 ** e), base):
            assert torch.equal(a, b * 2.0 ** e)


def _wcol(m, cin):
    """wcat column of row-split basis column m."""
    blk, c = divmod(m, cin + 32)
    return 96 + 4 * blk + c if c < cin else 32 * blk + c - cin


@pytest.mark.parametrize("graph", ["chickenpox", "metr_la"])
def test_row_split_vs_one_sm_kernel(graph):
    if graph == "chickenpox":
        ei, ew, _, _ = chickenpox_train_split()
        N = 20
    else:
        e, w, _ = synthetic.metr_la_like(0, 16)
        ei, ew, N = torch.from_numpy(e), torch.from_numpy(w), 207
    plan = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), N, "sym")
    for n_ops in (0, 1):
        for cin in (1, 4):
            assert ops.gru_seq_supported(plan, n_ops, cin, 32) and ops.gru_rows_supported(plan, n_ops, cin, 32)
            torch.manual_seed(10 * n_ops + cin)
            nb = (n_ops + 1) * (cin + 32)
            wcat = torch.zeros(96, 112, device=DEV)
            for k in range(n_ops + 1):
                wcat[:, 32 * k:32 * k + 32] = torch.randn(96, 32, device=DEV) * 0.15
                wcat[:, 96 + 4 * k:96 + 4 * k + cin] = torch.randn(96, cin, device=DEV) * 0.3
            bcat = torch.randn(96, device=DEV) * 0.1
            cols = [_wcol(m, cin) for m in range(nb)]
            wr = wcat[:, cols].contiguous()
            x = torch.randn(N, cin, device=DEV)
            h = torch.randn(N, 32, device=DEV) * 0.5
            gw = torch.randn(N, 32, device=DEV)
            for with_h in (True, False):
                res = []
                for rows in (True, False):
                    xl = x.clone().requires_grad_(True)
                    hl = h.clone().requires_grad_(True) if with_h else None
                    if rows:
                        wl, bl = wr.clone().requires_grad_(True), bcat.clone().requires_grad_(True)
                        out = ops.gru_rows_train(plan, n_ops, xl, hl, wl.detach(), bl.detach(), [("w", 0, 96, 0, nb), ("b", 0, 96)], [wl, bl])
                        assert torch.equal(out.detach(), ops.gru_rows_fwd(plan, n_ops, x, h if with_h else None, wr, bcat))
                    else:
                        wl, bl = wcat.clone().requires_grad_(True), bcat.clone().requires_grad_(True)
                        out = ops.gru_seq_train(plan, n_ops, xl.view(1, 1, N, cin), None if hl is None else hl.view(1, N, 32), wl.detach(),
                                                bl.detach(), None, [("w", 0, 96, 0, 112), ("b", 0, 96)], [wl, bl]).view(N, 32)
                    (out * gw).sum().backward()
                    res.append((out.detach(), xl.grad, hl.grad if with_h else None, wl.grad if rows else wl.grad[:, cols], bl.grad))
                (o1, *g1), (o2, *g2) = res
                _close(o1, o2)
                for a, b in zip(g1, g2):
                    assert (a is None) == (b is None)
                    if b is not None:
                        _close_grad(a, b)


def _random_graph(N, seed, deg=8):
    """Random weighted directed graph with a hub of 1200 in-edges (node 0), one of 1200 out-edges (node 1) and 17 isolated nodes."""
    g = torch.Generator().manual_seed(seed)
    live = N - 17
    src = torch.randint(0, live, (deg * live,), generator=g)
    dst = torch.randint(0, live, (deg * live,), generator=g)
    hub_in = torch.randperm(live, generator=g)[:1200]
    hub_out = torch.randperm(live, generator=g)[:1200]
    src = torch.cat([src, hub_in, torch.ones(1200, dtype=torch.long)])
    dst = torch.cat([dst, torch.zeros(1200, dtype=torch.long), hub_out])
    keep = src != dst
    ei = torch.stack([src[keep], dst[keep]])
    ei = torch.unique(ei, dim=1)
    ew = torch.rand(ei.size(1), generator=g) + 0.1
    return ei.to(DEV), ew.to(DEV)


@pytest.mark.parametrize("norm", ["sym", "rw", None])
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("cin", [1, 4, 5, 14, 16])
def test_fused_vs_autograd_on_random_graphs(cin, K, norm):
    N = 1000 + 389 * (cin % 5) + 7 * K                         # 1000..2600 nodes, never a multiple of the 16-row tile
    N += 1 if N % 16 == 0 else 0
    ei, ew = _random_graph(N, cin + 10 * K)
    lam = torch.tensor(1.7, device=DEV) if norm == "rw" else None
    for bias in (True, False):
        for with_h in (False, True):
            for x_grad in (False, True):
                m, X, H, w = _cell(cin, K, N, norm, bias, seed=cin + 10 * K)
                res = []
                for fused in (True, False):
                    m.fused_training = fused
                    m.zero_grad(set_to_none=True)
                    Xl = X.clone().requires_grad_(x_grad)
                    Hl = H.clone().requires_grad_(True) if with_h else None
                    c0 = _lib.path_counters()
                    out = m(Xl, ei, ew, Hl, lambda_max=lam)
                    (out * w).sum().backward()
                    assert _ran(c0, "k_gru_rows_bwd_a") == int(fused)
                    res.append([out.detach(), Xl.grad, None if Hl is None else Hl.grad] + [p.grad.clone() for p in m.parameters()])
                (of, *gf), (oa, *ga) = res
                _close(of, oa)
                for a, b in zip(gf, ga):
                    assert (a is None) == (b is None)
                    if b is not None:
                        _close_grad(a, b)


def test_fused_vs_autograd_on_a_50000_node_graph():
    N = 50000
    ei, ew = _random_graph(N, 7, deg=6)
    m, X, H, w = _cell(14, 2, N, "sym", True, seed=3)
    res = []
    for fused in (True, False):
        m.fused_training = fused
        m.zero_grad(set_to_none=True)
        Xl, Hl = X.clone().requires_grad_(True), H.clone().requires_grad_(True)
        out = m(Xl, ei, ew, Hl)
        (out * w).sum().backward()
        res.append([out.detach(), Xl.grad, Hl.grad] + [p.grad.clone() for p in m.parameters()])
    _close(res[0][0], res[1][0])
    for a, b in zip(res[0][1:], res[1][1:]):
        _close_grad(a, b)


def test_cuda_graph_replay_of_the_wikimaths_tutorial_step(golden_dir):
    """The tutorial's per-snapshot step (forward with H = None, MSE, backward, Adam(lr = 0.01)) captured once and replayed over the
    fixture's snapshots equals the same steps run eagerly."""
    g = load(golden_dir)
    c = g["cases"]["K2_sym"]
    ei, ew, X, Y = g["edge_index"].to(DEV).long(), g["edge_weight"].to(DEV), g["X"].to(DEV), g["Y"].to(DEV)
    m = model_for(c, DEV, True)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    xs, ys = X[0].clone(), Y[0].clone()

    def step():
        cost = torch.mean((m.linear(torch.relu(m.recurrent(xs, ei, ew))).squeeze() - ys) ** 2)
        cost.backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
        return cost

    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step()
    m.load_state_dict(c["state"])
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    replay = []
    for t in range(X.shape[0]):
        xs.copy_(X[t])
        ys.copy_(Y[t])
        graph.replay()
        replay.append(loss.detach().clone())
    torch.cuda.synchronize()
    m_e = model_for(c, DEV, True)
    opt_e = torch.optim.Adam(m_e.parameters(), lr=0.01)
    for t in range(X.shape[0]):
        cost = torch.mean((m_e.linear(torch.relu(m_e.recurrent(X[t], ei, ew))).squeeze() - Y[t]) ** 2)
        cost.backward()
        opt_e.step()
        opt_e.zero_grad()
        _close(replay[t], cost.detach(), 1e-5, 1e-7)
    for p, pe in zip(m.parameters(), m_e.parameters()):
        _close(p, pe, 1e-5, 1e-6)


def _ring(N):
    s = torch.arange(N, device=DEV)
    return torch.cat([torch.stack([s, (s + 1) % N]), torch.stack([(s + 1) % N, s])], dim=1)


def test_routing():
    """N > 207 with in_channels 17, K = 3, out_channels 16 or 3-D X stays op-for-op; graphs that fit one SM are served as before."""
    e300 = _ring(300)
    cases = [(GConvGRU(17, 32, 2), torch.randn(300, 17, device=DEV), torch.randn(300, 32, device=DEV)),
             (GConvGRU(4, 32, 3), torch.randn(300, 4, device=DEV), torch.randn(300, 32, device=DEV)),
             (GConvGRU(4, 16, 2), torch.randn(300, 4, device=DEV), torch.randn(300, 16, device=DEV)),
             (GConvGRU(4, 32, 2), torch.randn(2, 300, 4, device=DEV), torch.randn(2, 300, 32, device=DEV))]
    for mod, x, h in cases:
        mod = mod.to(DEV)
        for grad in (False, True):
            c0 = _lib.path_counters()
            with torch.set_grad_enabled(grad):
                mod(x, e300, None, h)
            assert all(_ran(c0, k) == 0 for k in ROWS)
    ei, ew, _, _ = chickenpox_train_split()
    ei, ew = ei.to(DEV), ew.to(DEV)
    for cin, kernel in ((4, "k_dcrnn_seq_tc"), (5, "k_spmm")):
        m = GConvGRU(cin, 32, 2).to(DEV)
        x, h = torch.randn(20, cin, device=DEV), torch.randn(20, 32, device=DEV).requires_grad_(True)
        c0 = _lib.path_counters()
        with torch.no_grad():
            m(x, ei, ew, h)
        m(x, ei, ew, h).sum().backward()
        assert _ran(c0, kernel) > 0 and all(_ran(c0, k) == 0 for k in ROWS)
    m = GConvGRU(4, 32, 2).to(DEV)                              # 208 nodes: the row-split path, never the one-SM backward
    c0 = _lib.path_counters()
    m(torch.randn(208, 4, device=DEV), _ring(208), None, torch.randn(208, 32, device=DEV).requires_grad_(True)).sum().backward()
    assert _ran(c0, "k_gru_rows_bwd_a") == 1 and _ran(c0, "k_gru_bwd_seq") == 0


def test_abi_errors():
    ei, ew, _, _ = chickenpox_train_split()
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 20, "sym")
    L = _lib.lib()
    h = cheb.handle
    buf = torch.zeros(1 << 20, device=DEV)
    p, q = _lib.ptr(buf), ctypes.c_void_p(buf.data_ptr() + 4)       # q: 4-byte aligned only
    r = ctypes.c_void_p(buf.data_ptr() + 2)                         # r: misaligned
    assert L.stmp_gru_rows_supported(h, 1, 16, 32) == 1 and L.stmp_gru_rows_supported(h, 0, 1, 32) == 1
    assert L.stmp_gru_rows_supported(h, 1, 17, 32) == 0 and L.stmp_gru_rows_supported(h, 2, 4, 32) == 0
    assert L.stmp_gru_rows_supported(h, 1, 4, 16) == 0 and L.stmp_gru_rows_supported(None, 1, 4, 32) == 0
    ld = ops.gru_rows_basis_ld(1, 4)
    fwd = lambda n_ops, cin, x=p, hh=p, S1=p, ldv=ld: L.stmp_gru_rows_fwd(h, n_ops, cin, x, hh, p, p, p, p, p, S1, p, ldv, None)
    assert fwd(1, 17) == _lib.STMP_EUNSUPPORTED and fwd(2, 4) == _lib.STMP_EUNSUPPORTED
    assert fwd(1, 4, x=None) == _lib.STMP_EINVAL
    assert fwd(1, 4, ldv=ld + 8) == _lib.STMP_ESHAPE and fwd(1, 4, x=r) == _lib.STMP_ESHAPE and fwd(1, 4, S1=q) == _lib.STMP_ESHAPE
    assert L.stmp_gru_rows_fwd(h, 1, 4, p, None, p, p, None, p, p, p, p, ld, None) == _lib.STMP_EINVAL      # S2 without h
    bwd = lambda cin, g=p, hh=p, dh=p: L.stmp_gru_rows_bwd(h, 1, cin, g, hh, p, p, p, p, p, p, dh, None)
    assert bwd(17) == _lib.STMP_EUNSUPPORTED and bwd(4, g=None) == _lib.STMP_EINVAL and bwd(4, hh=None) == _lib.STMP_EINVAL
    assert bwd(4, g=r) == _lib.STMP_ESHAPE
    wg = lambda n_ops, ldv, S1=p: L.stmp_gru_rows_wgrad(n_ops, 4, 20, ldv, S1, p, p, p, p, p, p, None)
    assert wg(1, ld + 8) == _lib.STMP_ESHAPE and wg(2, ld) == _lib.STMP_EUNSUPPORTED and wg(1, ld, S1=None) == _lib.STMP_EINVAL
    assert wg(1, ld, S1=q) == _lib.STMP_ESHAPE
    assert L.stmp_gru_rows_pack_weights(1, 17, p, p, None, None, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_gru_rows_pack_weights(1, 4, None, p, None, None, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_gru_rows_pack_weights(1, 4, p, p, p, None, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_gru_rows_wgrad_workspace_bytes(1, 16) > 0 and L.stmp_gru_rows_scratch_bytes(h) == 20 * 192 * 4
