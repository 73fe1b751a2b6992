"""GConvGRU training on the generic graph-GRU kernels: forward = `stmp_gru_seq_fwd` with a stash (the inference launch), backward =
`stmp_gru_pack_bwd_weights` -> `stmp_gru_bwd_basis` -> `stmp_gru_bwd_seq` -> `stmp_gru_bwd_wgrad`.  The reference's tutorial loop against
the unmodified reference (tests/golden/make_goldens_gconvgru.py), the fused path against the op-for-op autograd path
(`fused_training = False`), the ops-level entries with B > 1 windows of T > 1 steps on Chebyshev, GCN and DConv plans, and the C ABI."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU
from pytorch_geometric_temporal_b200.plan import GraphPlan
from gconvgru_seq import chickenpox_train_split, load, model_for, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDENS = [f"gconvgru_chickenpox_K{K}_{n}" for K in (1, 2) for n in ("sym", "rw", "carried")] + ["gconvgru_metr_la_K2"]
BWD_KERNELS = ("k_gru_pack_bwd_weights", "k_gru_bwd_basis", "k_gru_bwd_seq", "k_dcrnn_wgrad_tc", "k_gru_wgrad_reduce")


def _ran(before, name):
    return _lib.path_counters().get(name, 0) - before.get(name, 0)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _close_grad(got, want):
    _close(got, want, 1e-3, 1e-3 * want.abs().max().item() + 1e-6)


def _run_golden(g, fused):
    m = model_for(g, DEV, fused)
    H0 = g["H0"].to(DEV).requires_grad_(True) if "H0" in g else None
    c0 = _lib.path_counters()
    out, loss = run(m, g, DEV, H0)
    loss.backward()
    return m, H0, out, loss, c0


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", GOLDENS)
def test_training_vs_reference_golden(golden_dir, name, fused):
    g = load(golden_dir, name)
    m, H0, out, loss, c0 = _run_golden(g, fused)
    assert _ran(c0, "k_gru_bwd_seq") == (g["X"].shape[0] if fused else 0)
    _close(out, g["out"])
    _close(loss, g["loss"])
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        _close_grad(p.grad, g["grads"][k])
    if H0 is not None:
        _close_grad(H0.grad, g["gH0"])


def _chickenpox_graph():
    ei, ew, _, _ = chickenpox_train_split()
    return ei.to(DEV), ew.to(DEV)


def _cell(cin, K, norm="sym", bias=True, seed=0, N=20):
    torch.manual_seed(seed)
    m = GConvGRU(cin, 32, K, normalization=norm, bias=bias).to(DEV)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn_like(p) * 0.1)
    X = torch.randn(N, cin, device=DEV)
    H = torch.randn(N, 32, device=DEV) * 0.5
    w = torch.randn(N, 32, device=DEV)
    return m, X, H, w


def test_training_forward_is_bit_equal_to_inference_and_backward_is_deterministic():
    ei, ew = _chickenpox_graph()
    for K in (1, 2):
        m, X, H, w = _cell(3, K)
        c0 = _lib.path_counters()
        out = m(X, ei, ew, H)
        assert out.requires_grad and _ran(c0, "k_dcrnn_seq_tc") == 1
        with torch.no_grad():
            assert torch.equal(out.detach(), m(X, ei, ew, H))
            assert torch.equal(m(X, ei, ew), m(X, ei, ew, torch.zeros_like(H)))

        def grads():
            m.zero_grad(set_to_none=True)
            Xl, Hl = X.clone().requires_grad_(True), H.clone().requires_grad_(True)
            (m(Xl, ei, ew, Hl) * w).sum().backward()
            return [Xl.grad, Hl.grad] + [p.grad.clone() for p in m.parameters()]
        for a, b in zip(grads(), grads()):
            assert torch.equal(a, b)


@pytest.mark.parametrize("norm", ["sym", "rw", None])
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("cin", [1, 2, 3, 4])
def test_fused_vs_autograd(cin, K, norm):
    ei, ew = _chickenpox_graph()
    lam = torch.tensor(1.7, device=DEV) if norm == "rw" else None
    for bias in (True, False):
        for h_mode in ("none", "leaf", "carried"):
            for x_grad in (False, True):
                m, X, H, w = _cell(cin, K, norm, bias, seed=cin + 10 * K)
                res = []
                for fused in (True, False):
                    m.fused_training = fused
                    m.zero_grad(set_to_none=True)
                    Xl = X.clone().requires_grad_(x_grad)
                    Hl = H.clone().requires_grad_(True) if h_mode != "none" else None
                    c0 = _lib.path_counters()
                    h = m(Xl, ei, ew, Hl, lambda_max=lam)
                    if h_mode == "carried":
                        h = m(Xl * 0.5, ei, ew, h, lambda_max=lam)
                    (h * w).sum().backward()
                    assert _ran(c0, "k_gru_bwd_seq") == (1 + (h_mode == "carried")) * fused
                    res.append((h.detach(), Xl.grad, None if Hl is None else Hl.grad, [p.grad.clone() for p in m.parameters()]))
                (of, xf, hf, gf), (oa, xa, ha, ga) = res
                _close(of, oa)
                assert (xf is None) == (not x_grad) and (hf is None) == (h_mode == "none")
                for a, b in zip([xf, hf] + gf, [xa, ha] + ga):
                    if b is not None:
                        _close_grad(a, b)


def _restated(plan, n_ops, x, h0, wcat, bcat, spmm=None, stash=None):
    """The recurrence of stmp_gru_seq_fwd chained op for op from differentiable SpMMs and torch ops.  `spmm(k, t)` applies operator k
    (default: the plan's, `ops.spmm`); h0 (B, N, 32), or one (N, 32) state shared by every window.  A `stash` list receives the
    kernel's stash of every step, (Z, R, H~)."""
    B, T, N, Ci = x.shape
    H = x.new_zeros(B, N, 32) if h0 is None else h0.expand(B, N, 32)
    spmm = spmm or (lambda k, t: ops.spmm(plan, k, t))

    def A(X, Hp):
        cols = [Hp] + [spmm(k, Hp) for k in range(n_ops)] + [Hp.new_zeros(B, N, 32)] * (2 - n_ops)
        xs = [X] + [spmm(k, X) for k in range(n_ops)] + [X.new_zeros(B, N, Ci)] * (2 - n_ops)
        pad = [X.new_zeros(B, N, 4 - Ci)] * 3
        xcols = [t for pair in zip(xs, pad) for t in pair]
        return torch.cat(cols + xcols + [X.new_zeros(B, N, 4)], dim=-1)
    outs = []
    for t in range(T):
        pre = A(x[:, t], H) @ wcat.t() + bcat
        Z, R = torch.sigmoid(pre[..., :32]), torch.sigmoid(pre[..., 32:64])
        Ht = torch.tanh((A(x[:, t], H * R) @ wcat.t() + bcat)[..., 64:])
        if stash is not None:
            stash.append((Z, R, Ht))
        H = Z * H + (1 - Z) * Ht
        outs.append(H)
    return torch.stack(outs, dim=1)


@pytest.mark.parametrize("flavor,n_ops", [("cheb", 0), ("cheb", 1), ("gcn", 1), ("dconv", 1), ("dconv", 2)])
def test_ops_level_windows_and_steps_vs_autograd(flavor, n_ops):
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    N = 207
    plan = {"cheb": lambda: GraphPlan(_lib.FLAVOR_CHEB, ei, ew, N, "sym"), "gcn": lambda: GraphPlan(_lib.FLAVOR_GCN, ei, ew, N),
            "dconv": lambda: GraphPlan(_lib.FLAVOR_DCONV, ei, ew, N, flags=_lib.DCONV_ALLOW_DUPLICATES)}[flavor]()
    torch.manual_seed(n_ops)
    B, T, Ci = 3, 4, 3
    assert ops.gru_bwd_supported(plan, n_ops, Ci, 32) and ops.gru_seq_supported(plan, n_ops, Ci, 32)
    wcat = torch.zeros(96, 112, device=DEV)
    for k in range(n_ops + 1):
        wcat[:, 32 * k:32 * k + 32] = torch.randn(96, 32, device=DEV) * 0.15
        wcat[:, 96 + 4 * k:96 + 4 * k + Ci] = torch.randn(96, Ci, device=DEV) * 0.3
    bcat = torch.randn(96, device=DEV) * 0.1
    x = torch.randn(B, T, N, Ci, device=DEV)
    h0 = torch.randn(B, N, 32, device=DEV) * 0.5
    w = torch.randn(B, T, N, 32, device=DEV)
    spec = [("w", 0, 96, 0, 112), ("b", 0, 96)]
    res = []
    for fused in (True, False):
        xl, hl = x.clone().requires_grad_(True), h0.clone().requires_grad_(True)
        wl, bl = wcat.clone().requires_grad_(True), bcat.clone().requires_grad_(True)
        c0 = _lib.path_counters()
        if fused:
            out = ops.gru_seq_train(plan, n_ops, xl, hl, wl.detach(), bl.detach(), None, spec, [wl, bl])
        else:
            out = _restated(plan, n_ops, xl, hl, wl, bl)
        (out * w).sum().backward()
        assert _ran(c0, "k_gru_bwd_seq") == int(fused)
        res.append([out.detach(), xl.grad, hl.grad, wl.grad, bl.grad])
    _close(res[0][0], res[1][0])
    for a, b in zip(res[0][1:], res[1][1:]):
        _close_grad(a, b)
    live = torch.zeros(96, 112, dtype=torch.bool)
    for k in range(n_ops + 1):
        live[:, 32 * k:32 * k + 32] = True
        live[:, 96 + 4 * k:96 + 4 * k + Ci] = True
    assert torch.all(res[0][3].cpu()[~live] == 0)                 # absent operators, channels and the padding


def test_path_counters_and_launches_of_one_training_call():
    ei, ew = _chickenpox_graph()
    m, X, H, w = _cell(4, 2)
    Hl = H.clone().requires_grad_(True)
    (m(X, ei, ew, Hl) * w).sum().backward()                       # warm: plan, packed weights, workspaces
    c0, n0 = _lib.path_counters(), _lib.launch_count()
    (m(X, ei, ew, Hl) * w).sum().backward()
    assert _lib.launch_count() - n0 == 1 + len(BWD_KERNELS)
    assert {k: _ran(c0, k) for k in ("k_dcrnn_seq_tc", "k_spmm") + BWD_KERNELS} == {
        "k_dcrnn_seq_tc": 1, "k_spmm": 0, **{k: 1 for k in BWD_KERNELS}}


@pytest.mark.parametrize("name", ["gconvgru_chickenpox_K2_carried", "gconvgru_chickenpox_K1_sym"])
def test_gradients_scale_with_a_power_of_two_loss_scale_bit_for_bit(golden_dir, name):
    g = load(golden_dir, name)

    def grads(scale):
        m = model_for(g, DEV, True)
        H0 = g["H0"].to(DEV).requires_grad_(True) if "H0" in g else None
        c0 = _lib.path_counters()
        _, loss = run(m, g, DEV, H0)
        (loss * scale).backward()
        assert _ran(c0, "k_gru_bwd_seq") == g["X"].shape[0]
        return [p.grad for p in m.parameters()] + ([H0.grad] if H0 is not None else [])
    base = grads(1.0)
    for e in (-24, 8):
        for a, b in zip(grads(2.0 ** e), base):
            assert torch.equal(a, b * 2.0 ** e)


def test_cuda_graph_replay_of_a_chickenpox_epoch(golden_dir):
    """examples/recurrent/gconvgru_example.py's epoch (forward over the train split with H = None, one backward, Adam) as one CUDA graph."""
    g = load(golden_dir, "gconvgru_chickenpox_K2_sym")
    g = {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in g.items()}
    m = model_for(g, DEV, True)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    state0 = {k: v.clone() for k, v in m.state_dict().items()}

    def epoch():
        opt.zero_grad(set_to_none=False)
        _, loss = run(m, g, DEV)
        loss.backward()
        opt.step()
        return loss

    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            epoch()
    torch.cuda.current_stream().wait_stream(side)
    m_e = model_for(g, DEV, True)
    m_e.load_state_dict(state0)
    opt_e = torch.optim.Adam(m_e.parameters(), lr=0.01)
    eager = []
    for _ in range(2):
        opt_e.zero_grad()
        _, le = run(m_e, g, DEV)
        le.backward()
        opt_e.step()
        eager.append(le.detach())
    m.load_state_dict(state0)
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = epoch()
    m.load_state_dict(state0)
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    replay = []
    for _ in range(2):
        graph.replay()
        replay.append(loss.detach().clone())
    torch.cuda.synchronize()
    for a, b in zip(replay, eager):
        _close(a, b, 1e-5, 1e-7)
    for p, pe in zip(m.parameters(), m_e.parameters()):
        _close(p, pe, 1e-5, 1e-6)


def _ring(N):
    s = torch.arange(N, device=DEV)
    return torch.cat([torch.stack([s, (s + 1) % N]), torch.stack([(s + 1) % N, s])], dim=1), None


def test_routing_at_the_envelope_edges():
    """N = 208 (above the fused kernels' 207 nodes), K = 3, out_channels = 16 and 3-D X stay on the op-for-op path and still train."""
    ei, ew = _chickenpox_graph()
    e208, _ = _ring(208)
    m, X, H, w = _cell(4, 2)
    cases = [(GConvGRU(4, 32, 2), torch.randn(208, 4, device=DEV), e208, None, torch.randn(208, 32, device=DEV)),
             (GConvGRU(4, 32, 3), X, ei, ew, H), (GConvGRU(4, 16, 2), X, ei, ew, H[:, :16]),
             (GConvGRU(4, 32, 2), X.expand(2, 20, 4), ei, ew, H.expand(2, 20, 32))]
    for mod, x, e, wgt, h in cases:
        mod = mod.to(DEV)
        c0 = _lib.path_counters()
        xl, hl = x.clone().requires_grad_(True), h.clone().requires_grad_(True)
        out = mod(xl, e, wgt, hl)
        out.square().sum().backward()
        assert _ran(c0, "k_gru_bwd_seq") == 0
        ref = GConvGRU(mod.in_channels, mod.out_channels, mod.K).to(DEV)
        ref.load_state_dict(mod.state_dict())
        ref.fused_training = False
        xr, hr = x.clone().requires_grad_(True), h.clone().requires_grad_(True)
        ref(xr, e, wgt, hr).square().sum().backward()
        _close_grad(xl.grad, xr.grad)
        _close_grad(hl.grad, hr.grad)
    # a non-contiguous H is served by the fused path
    Hnc = H.t().contiguous().t().requires_grad_(True)
    assert not Hnc.is_contiguous()
    c0 = _lib.path_counters()
    (m(X, ei, ew, Hnc) * w).sum().backward()
    assert _ran(c0, "k_gru_bwd_seq") == 1


def test_abi_errors():
    ei, ew = _chickenpox_graph()
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei, ew, 20, "sym")
    L = _lib.lib()
    buf = torch.zeros(1 << 20, device=DEV)
    p, q = _lib.ptr(buf), __import__("ctypes").c_void_p(buf.data_ptr() + 4)     # q: 4-byte aligned only
    h = cheb.handle
    assert L.stmp_gru_bwd_supported(h, 1, 4, 32) == 1 and L.stmp_gru_bwd_supported(h, 0, 1, 32) == 1
    assert L.stmp_gru_bwd_supported(h, 2, 4, 32) == 0 and L.stmp_gru_bwd_supported(h, 1, 4, 16) == 0
    assert L.stmp_gru_bwd_supported(h, 1, 5, 32) == 0 and L.stmp_gru_bwd_supported(None, 1, 4, 32) == 0
    ld = ops.gru_bwd_basis_ld(1, 4)
    seq = lambda n_ops, B, T, cin, gout, h0, hs, stash=p: L.stmp_gru_bwd_seq(h, n_ops, B, T, cin, gout, p, h0, hs, stash, p, p, p, p, None, p,
                                                                             None)
    assert seq(2, 1, 1, 4, p, None, 0) == _lib.STMP_EUNSUPPORTED                 # more operators than the plan has
    assert seq(1, 1, 1, 5, p, None, 0) == _lib.STMP_EUNSUPPORTED                 # cin outside 1..4
    assert seq(1, 2, 1, 4, p, p, 0) == _lib.STMP_EUNSUPPORTED                    # a shared h0
    assert seq(1, 1, 1, 4, None, None, 0) == _lib.STMP_EINVAL
    assert seq(1, 1, 0, 4, p, None, 0) == _lib.STMP_ESHAPE
    assert seq(1, 1, 1, 4, p, p, 7) == _lib.STMP_ESHAPE                          # h0 not (B, N, 32) dense
    assert seq(1, 1, 1, 4, q, None, 0) == _lib.STMP_ESHAPE                       # misaligned
    basis = lambda ldv, x=p, hs=20 * 32: L.stmp_gru_bwd_basis(h, 1, 1, 1, 4, x, 80, 80, p, p, hs, p, p, p, ldv, None)
    assert basis(ld + 8) == _lib.STMP_ESHAPE and basis(ld, x=None) == _lib.STMP_EINVAL and basis(ld, hs=0) == _lib.STMP_EUNSUPPORTED
    wg = lambda n_ops, ldv, S1=p: L.stmp_gru_bwd_wgrad(n_ops, 4, 20, ldv, S1, p, p, p, p, p, p, None)
    assert wg(1, ld + 8) == _lib.STMP_ESHAPE and wg(3, ld) == _lib.STMP_EUNSUPPORTED and wg(1, ld, S1=None) == _lib.STMP_EINVAL
    assert L.stmp_gru_pack_bwd_weights(1, 5, p, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_gru_pack_bwd_weights(1, 4, None, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_gru_bwd_wgrad_workspace_bytes(1, 4) > 0
