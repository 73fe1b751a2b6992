"""GConvLSTM and GCLSTM at 32 hidden channels on the row-split LSTM cell kernel (`stmp_lstm_rows_*`, DESIGN §4j): the reference's chickenpox
tutorial epochs, a METR-LA-shaped carried sequence and WikiMaths snapshots against the unmodified reference (tests/golden/make_goldens_lstm.py),
fused and op-for-op; launch counts; bit-equality of training and inference forwards; determinism and loss-scale equivariance of the
backward; structurally zero gradients; the fused path against op-for-op autograd on random graphs with hubs and isolated nodes; a captured
tutorial epoch; routing; and the C ABI's errors."""
import ctypes

import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvLSTM
from pytorch_geometric_temporal_b200.plan import GraphPlan
from gconvgru_seq import chickenpox_train_split
import lstm_seq

pytestmark = pytest.mark.gpu
DEV = "cuda"
DATA = ["chickenpox_K1_sym", "chickenpox_K2_sym", "chickenpox_K2_rw", "metr_la_K2", "wikimaths_K2"]
CASES = [f"{m}_{d}" for m in ("gconvlstm", "gclstm") for d in DATA]
ROWS = ("k_lstm_rows_fwd", "k_lstm_rows_bwd_a", "k_lstm_rows_bwd_b", "k_lstm_rows_wgrad_reduce")


def _ran(before, name):
    return _lib.path_counters().get(name, 0) - before.get(name, 0)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _close_grad(got, want):
    _close(got, want, 1e-3, 1e-5)


@pytest.fixture(scope="module")
def goldens(golden_dir):
    return lstm_seq.load(golden_dir)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", CASES)
def test_vs_reference_golden(golden_dir, goldens, case, fused):
    c = goldens["cases"][case]
    m = lstm_seq.model_for(goldens, case, DEV, fused)
    c0 = _lib.path_counters()
    out, cost, H0, C0 = lstm_seq.run_case(m, goldens, case, golden_dir, DEV)
    cost.backward()
    S = out.shape[0]
    if fused:
        assert _ran(c0, "k_lstm_rows_fwd") == S and _ran(c0, "k_lstm_rows_bwd_a") == S
        assert _ran(c0, "k_spmm") == 0 and _ran(c0, "k_gemm_split") == 0
        assert _ran(c0, "k_lstm_rows_bwd_b") == (S - (H0 is None) if c["K"] == 2 else 0)   # step 0 from H = None has no dH
    else:
        assert all(_ran(c0, k) == 0 for k in ROWS)
    _close(out, c["out"])
    _close(cost, c["loss"])
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        _close_grad(p.grad, c["grads"][k])
    if H0 is not None:
        _close_grad(H0.grad, c["gH0"])
        _close_grad(C0.grad, c["gC0"])


def _ring(N):
    s = torch.arange(N, device=DEV)
    return torch.cat([torch.stack([s, (s + 1) % N]), torch.stack([(s + 5) % N, s])], dim=1)


def _cell(cls, cin, K, N, norm="sym", bias=True, seed=0):
    torch.manual_seed(seed)
    m = cls(cin, 32, K, normalization=norm, bias=bias).to(DEV)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("bias") or n.startswith("b_"):
                p.copy_(torch.randn_like(p) * 0.1)
    return (m, torch.randn(N, cin, device=DEV), torch.randn(N, 32, device=DEV) * 0.5, torch.randn(N, 32, device=DEV),
            torch.randn(N, 32, device=DEV), torch.randn(N, 32, device=DEV))


@pytest.mark.parametrize("cls", [GConvLSTM, GCLSTM])
def test_launch_counts(cls):
    N = 1068
    e = _ring(N)
    for K in (1, 2):
        m, x, H, C, wh, wc = _cell(cls, 14, K, N, seed=K)
        xw, Hw, Cw = (t.clone().requires_grad_(True) for t in (x, H, C))
        sum(t.sum() for t in m(xw, e, None, Hw, Cw)).backward()      # warm: plan, packed weights, workspaces
        with torch.no_grad():
            m.b_i.add_(0.01)
            n0 = _lib.launch_count()
            m(x, e, None, H, C)
            assert _lib.launch_count() - n0 == 2                       # a parameter changed: one pack, then the cell
            n0 = _lib.launch_count()
            m(x, e, None, H, C)
            m(x, e, None)
            assert _lib.launch_count() - n0 == 2                       # one launch per call
        for need_x, need_state in ((False, False), (True, False), (False, True), (True, True)):
            xl = x.clone().requires_grad_(need_x)
            Hl, Cl = H.clone().requires_grad_(need_state), C.clone().requires_grad_(need_state)
            n0 = _lib.launch_count()
            hn, cn = m(xl, e, None, Hl, Cl)
            assert _lib.launch_count() - n0 == 1
            loss = (hn * wh).sum() + (cn * wc).sum()
            c0, n0 = _lib.path_counters(), _lib.launch_count()
            loss.backward()
            gather = K == 2 and (need_state or (need_x and cls is GConvLSTM))
            assert _lib.launch_count() - n0 == 3 + gather              # rowwise, [gather], weight-gradient contraction + reduce
            assert {k: _ran(c0, k) for k in ROWS[1:] + ("k_dcrnn_wgrad", "k_spmm")} == {
                "k_lstm_rows_bwd_a": 1, "k_lstm_rows_bwd_b": int(gather), "k_lstm_rows_wgrad_reduce": 1, "k_dcrnn_wgrad": 1, "k_spmm": 0}


@pytest.mark.parametrize("cls", [GConvLSTM, GCLSTM])
def test_training_forward_is_bit_equal_to_inference_and_backward_is_deterministic(cls):
    N = 1500
    e = _ring(N)
    for K in (1, 2):
        m, x, H, C, wh, wc = _cell(cls, 5, K, N, seed=K)
        for h, c in ((H, C), (None, None), (H, None), (None, C)):
            hn, cn = m(x, e, None, h, c)
            assert hn.requires_grad
            with torch.no_grad():
                hi, ci = m(x, e, None, h, c)
            assert torch.equal(hn.detach(), hi) and torch.equal(cn.detach(), ci)

            def grads():
                m.zero_grad(set_to_none=True)
                xl = x.clone().requires_grad_(True)
                hl = None if h is None else h.clone().requires_grad_(True)
                cl = None if c is None else c.clone().requires_grad_(True)
                a, b = m(xl, e, None, hl, cl)
                ((a * wh).sum() + (b * wc).sum()).backward()
                return [xl.grad] + [t.grad for t in (hl, cl) if t is not None] + [p.grad.clone() for p in m.parameters()]
            for a, b in zip(grads(), grads()):
                assert torch.equal(a, b)


@pytest.mark.parametrize("case", ["gconvlstm_chickenpox_K2_sym", "gclstm_metr_la_K2", "gconvlstm_wikimaths_K2"])
def test_gradients_scale_with_a_power_of_two_loss_scale_bit_for_bit(golden_dir, goldens, case):
    def grads(scale):
        m = lstm_seq.model_for(goldens, case, DEV, True)
        c0 = _lib.path_counters()
        out, cost, H0, C0 = lstm_seq.run_case(m, goldens, case, golden_dir, DEV)
        (cost * scale).backward()
        assert _ran(c0, "k_lstm_rows_bwd_a") == out.shape[0]
        return [p.grad for p in m.parameters()] + ([H0.grad, C0.grad] if H0 is not None else [])
    base = grads(1.0)
    for e in (-24, 8):
        for a, b in zip(grads(2.0 ** e), base):
            assert torch.equal(a, b * 2.0 ** e)


@pytest.mark.parametrize("cls", [GConvLSTM, GCLSTM])
def test_structurally_zero_gradients_are_exact_zeros(cls):
    """One step from H = None: every H-column weight gets an exact zero gradient; from C = None the forget gate only scales a zero state,
    so every parameter of that gate and w_c_i get exact zeros too."""
    N = 700
    e = _ring(N)
    for K in (1, 2):
        m, x, H, C, wh, wc = _cell(cls, 4, K, N, seed=5 + K)
        for h, c in ((None, C), (H, None), (None, None)):
            m.zero_grad(set_to_none=True)
            a, b = m(x, e, None, h, c)
            ((a * wh).sum() + (b * wc).sum()).backward()
            for k, p in m.named_parameters():
                h_weight = (k.startswith("conv_h_") if cls is GConvLSTM else k.startswith("conv_")) and ".lins." in k
                f_gate = k.split(".")[0] in ("conv_x_f", "conv_h_f", "conv_f", "W_f", "b_f", "w_c_f")
                if (h is None and h_weight) or (c is None and (f_gate or k == "w_c_i")):
                    assert torch.all(p.grad == 0), k
                else:
                    assert p.grad.abs().sum() > 0, k


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
    ei = torch.unique(torch.stack([src[keep], dst[keep]]), dim=1)
    ew = torch.rand(ei.size(1), generator=g) + 0.1
    return ei.to(DEV), ew.to(DEV)


def _fused_vs_autograd(m, ei, ew, X, H, C, wh, wc, with_h, with_c, x_grad, lam=None):
    res = []
    for fused in (True, False):
        m.fused_training = fused
        m.zero_grad(set_to_none=True)
        Xl = X.clone().requires_grad_(x_grad)
        Hl = H.clone().requires_grad_(True) if with_h else None
        Cl = C.clone().requires_grad_(True) if with_c else None
        c0 = _lib.path_counters()
        a, b = m(Xl, ei, ew, Hl, Cl, lambda_max=lam)
        ((a * wh).sum() + (b * wc).sum()).backward()
        assert _ran(c0, "k_lstm_rows_bwd_a") == int(fused)
        res.append([a.detach(), b.detach(), Xl.grad] + [None if t is None else t.grad for t in (Hl, Cl)]
                   + [p.grad.clone() for p in m.parameters()])
    (hf, cf, *gf), (ha, ca, *ga) = res
    _close(hf, ha)
    _close(cf, ca)
    for a, b in zip(gf, ga):
        assert (a is None) == (b is None)
        if b is not None:
            _close(a, b, 1e-3, 1e-3 * b.abs().max().item() + 1e-6)


@pytest.mark.parametrize("cls", [GConvLSTM, GCLSTM])
@pytest.mark.parametrize("norm", ["sym", "rw", None])
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("cin", [1, 4, 5, 14, 16])
def test_fused_vs_autograd_on_random_graphs(cin, K, norm, cls):
    N = 1000 + 389 * (cin % 5) + 7 * K                         # 1000..2600 nodes, never a multiple of the 16-row tile
    N += 1 if N % 16 == 0 else 0
    ei, ew = _random_graph(N, cin + 10 * K)
    lam = torch.tensor(1.7, device=DEV) if norm == "rw" else None
    for bias in (True, False):
        for with_h, with_c in ((False, False), (True, True), (True, False), (False, True)):
            for x_grad in (False, True):
                m, X, H, C, wh, wc = _cell(cls, cin, K, N, norm, bias, seed=cin + 10 * K)
                _fused_vs_autograd(m, ei, ew, X, H, C, wh, wc, with_h, with_c, x_grad, lam)


@pytest.mark.parametrize("cls", [GConvLSTM, GCLSTM])
def test_fused_vs_autograd_on_a_50000_node_graph(cls):
    N = 50000
    ei, ew = _random_graph(N, 7, deg=6)
    m, X, H, C, wh, wc = _cell(cls, 14, 2, N, "sym", True, seed=3)
    _fused_vs_autograd(m, ei, ew, X, H, C, wh, wc, True, True, True)


@pytest.mark.parametrize("case", ["gconvlstm_chickenpox_K1_sym", "gclstm_chickenpox_K1_sym"])
def test_cuda_graph_replay_of_the_tutorial_epoch(golden_dir, goldens, case):
    """The tutorial's epoch (103 snapshots with H and C carried from None, cumulative MSE, one backward, Adam(lr = 0.01)) captured once
    and replayed for three epochs equals the same epochs run eagerly."""
    ei, ew, X, Y, _, _ = lstm_seq.data("chickenpox", golden_dir)
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV)
    m = lstm_seq.model_for(goldens, case, DEV, True)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)

    def epoch(model, o):
        _, cost = lstm_seq.run(model, ei, ew, X, Y, device=DEV)
        cost.backward()
        o.step()
        o.zero_grad(set_to_none=False)
        return cost

    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            epoch(m, opt)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = epoch(m, opt)
    m.load_state_dict(goldens["states"][goldens["cases"][case]["state"]])
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    c0 = _lib.path_counters()
    replay = []
    for _ in range(3):
        graph.replay()
        replay.append(loss.detach().clone())
    torch.cuda.synchronize()
    assert _ran(c0, "k_lstm_rows_fwd") == 0                      # replays launch no library call from the host
    m_e = lstm_seq.model_for(goldens, case, DEV, True)
    opt_e = torch.optim.Adam(m_e.parameters(), lr=0.01, capturable=True)     # the same update arithmetic as the captured optimiser
    for t in range(3):
        cost = epoch(m_e, opt_e)
        _close(replay[t], cost.detach(), 1e-5, 1e-7)
    _close(replay[0], goldens["cases"][case]["loss"])
    for p, pe in zip(m.parameters(), m_e.parameters()):
        _close(p, pe, 1e-5, 1e-6)


def test_routing(golden_dir):
    """In-envelope calls take the row-split kernel; cfg5's GConvLSTM(64, 64, 3) still trains through _LstmCellFn; out_channels 16, K = 3,
    in_channels 17 and 3-D X are unchanged."""
    e300 = _ring(300)
    for cls in (GConvLSTM, GCLSTM):
        for mod, x, h in ((cls(4, 32, 3), torch.randn(300, 4, device=DEV), torch.randn(300, 32, device=DEV)),
                          (cls(4, 16, 2), torch.randn(300, 4, device=DEV), torch.randn(300, 16, device=DEV)),
                          (cls(17, 32, 2), torch.randn(300, 17, device=DEV), torch.randn(300, 32, device=DEV)),
                          (cls(4, 32, 2), torch.randn(2, 300, 4, device=DEV), torch.randn(2, 300, 32, device=DEV))):
            mod = mod.to(DEV)
            for grad in (False, True):
                c0 = _lib.path_counters()
                with torch.set_grad_enabled(grad):
                    a, b = mod(x, e300, None, h, h)
                if grad:
                    (a.sum() + b.sum()).backward()
                assert all(_ran(c0, k) == 0 for k in ROWS)
        mod = cls(4, 32, 2).to(DEV)
        c0 = _lib.path_counters()
        with torch.no_grad():
            mod(torch.randn(300, 4, device=DEV), e300)
        a, b = mod(torch.randn(300, 4, device=DEV), e300)
        (a.sum() + b.sum()).backward()
        assert _ran(c0, "k_lstm_rows_fwd") == 2 and _ran(c0, "k_lstm_rows_bwd_a") == 1 and _ran(c0, "k_spmm") == 0
    cell = GConvLSTM(64, 64, 3).to(DEV)                         # cfg5's cell
    ei = torch.randint(0, 2000, (2, 20000), device=DEV)
    c0 = _lib.path_counters()
    a, b = cell(torch.randn(2000, 64, device=DEV), ei)
    (a.square().mean() + b.square().mean()).backward()
    assert _ran(c0, "k_lstm_gate_bwd") == 1 and all(_ran(c0, k) == 0 for k in ROWS)


def test_abi_errors():
    ei, ew, _, _ = chickenpox_train_split()
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 20, "sym")
    L = _lib.lib()
    h = cheb.handle
    GCV, GC = _lib.LSTM_GCONV, _lib.LSTM_GC
    buf = torch.zeros(1 << 20, device=DEV)
    p, q = _lib.ptr(buf), ctypes.c_void_p(buf.data_ptr() + 4)       # q: 4-byte aligned only
    r = ctypes.c_void_p(buf.data_ptr() + 2)                         # r: misaligned
    for v in (GCV, GC):
        assert L.stmp_lstm_rows_supported(h, v, 1, 16, 32) == 1 and L.stmp_lstm_rows_supported(h, v, 0, 1, 32) == 1
        assert L.stmp_lstm_rows_supported(h, v, 1, 17, 32) == 0 and L.stmp_lstm_rows_supported(h, v, 2, 4, 32) == 0
        assert L.stmp_lstm_rows_supported(h, v, 1, 4, 16) == 0 and L.stmp_lstm_rows_supported(None, v, 1, 4, 32) == 0
    assert L.stmp_lstm_rows_supported(h, 2, 1, 4, 32) == 0
    ld = ops.lstm_rows_basis_ld(GCV, 1, 4)
    assert ld == 72 and ops.lstm_rows_basis_ld(GC, 1, 4) == 72 and ops.lstm_rows_basis_ld(GC, 1, 5) == 72

    def fwd(n_ops=1, cin=4, v=GCV, x=p, S=p, ldv=ld):
        return L.stmp_lstm_rows_fwd(h, v, n_ops, cin, x, p, p, p, p, p, p, p, p, S, ldv, None)
    assert fwd(cin=17) == _lib.STMP_EUNSUPPORTED and fwd(n_ops=2) == _lib.STMP_EUNSUPPORTED and fwd(v=2) == _lib.STMP_EINVAL
    assert fwd(x=None) == _lib.STMP_EINVAL
    assert fwd(ldv=ld + 8) == _lib.STMP_ESHAPE and fwd(x=r) == _lib.STMP_ESHAPE and fwd(S=q) == _lib.STMP_ESHAPE

    def bwd(cin=4, cn=p, c=p, dc=p, dpre=p):
        return L.stmp_lstm_rows_bwd(h, GCV, 1, cin, p, p, c, cn, p, p, p, p, dpre, p, p, dc, None)
    assert bwd(cin=17) == _lib.STMP_EUNSUPPORTED and bwd(cn=None) == _lib.STMP_EINVAL and bwd(c=None) == _lib.STMP_EINVAL
    assert bwd(cn=r) == _lib.STMP_ESHAPE and bwd(dpre=q) == _lib.STMP_ESHAPE

    def wg(n_ops=1, ldv=ld, S=p, scratch=p, dpeep=p):
        return L.stmp_lstm_rows_wgrad(GCV, n_ops, 4, 20, ldv, S, p, scratch, p, p, p, dpeep, None)
    assert wg(ldv=ld + 8) == _lib.STMP_ESHAPE and wg(n_ops=2) == _lib.STMP_EUNSUPPORTED and wg(S=None) == _lib.STMP_EINVAL
    assert wg(S=q) == _lib.STMP_ESHAPE and wg(scratch=None) == _lib.STMP_EINVAL
    assert L.stmp_lstm_rows_pack_weights(GCV, 1, 17, p, p, None, None, p, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_lstm_rows_pack_weights(GCV, 1, 4, None, p, None, None, p, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_lstm_rows_pack_weights(GCV, 1, 4, p, p, p, None, p, p, p, None) == _lib.STMP_EINVAL     # one conv bias stack
    assert L.stmp_lstm_rows_pack_weights(GC, 1, 4, p, p, p, p, p, p, p, None) == _lib.STMP_EINVAL         # GCLSTM has no bx
    assert L.stmp_lstm_rows_wgrad_workspace_bytes(GCV, 1, 16) > 0 and L.stmp_lstm_rows_wgrad_workspace_bytes(GCV, 1, 17) == 0
    assert L.stmp_lstm_rows_scratch_bytes(h) == (20 * 48 + 2 * 96) * 4             # 20 rows: two 16-row tiles of peephole sums
    torch.cuda.synchronize()
