"""Host side of GConvGRU on the row-split cell kernels (stmp_gru_rows_*): the routing of a call (`GConvGRU._rows_ok`), the weight pack
(`GConvGRU._rows_packed`), the autograd Function `ops._GruRowsFn` and the hand-off of the packed weights' gradients to the parameters
(`GConvGRU._param_spec(rows=True)`, `ops._spec_grads`), with every library call replaced by a dense torch restatement of its contract on a
dense Chebyshev plan -- outputs, costs and EVERY gradient against the unmodified reference on WikiMaths
(tests/golden/make_goldens_wikimaths.py)."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU
from test_modules_host_logic_cpu import dense_graph_ops  # noqa: F401  (dense Chebyshev plan + SpMM, one-SM inference off)
from wikimaths_seq import load, model_for, run

CASES = ["K2_sym", "K1_sym", "K2_sym_carried", "K2_rw"]


def _basis(plan, n_ops, U):
    return torch.cat([U] + [torch.matmul(plan.L, U)] * n_ops, dim=-1)


def _adjoint(plan, n_ops, dS, C):
    dU = dS[..., :C].clone()
    if n_ops:
        dU += torch.matmul(plan.L.t(), dS[..., C:2 * C])
    return dU


def fake_pack(n_ops, cin, wx, wh, bx=None, bh=None):
    C = cin + 32
    w = wx.new_zeros(96, (n_ops + 1) * C)
    for g in range(3):
        for k in range(n_ops + 1):
            w[32 * g:32 * g + 32, k * C:k * C + cin] = wx[g, k]
            w[32 * g:32 * g + 32, k * C + cin:(k + 1) * C] = wh[g, k]
    return w, ((bx + bh).reshape(96) if bx is not None else wx.new_zeros(96))


def fake_fwd(plan, n_ops, x, h, w, b, train=False):
    H = x.new_zeros(x.size(0), 32) if h is None else h
    S1 = _basis(plan, n_ops, torch.cat([x, H], -1))
    pre = S1 @ w.t() + b
    Z, R = torch.sigmoid(pre[:, :32]), torch.sigmoid(pre[:, 32:64])
    S2 = _basis(plan, n_ops, torch.cat([x, H * R], -1))
    Ht = torch.tanh((S2 @ w.t() + b)[:, 64:])
    out = Z * H + (1 - Z) * Ht
    return (out, torch.stack([Z, R, Ht]), S1, S2) if train else out


def fake_bwd(plan, n_ops, gout, h, stash, w, want_dx, want_dh, cin):
    Z, R, Ht = stash
    C = cin + 32
    Hp = torch.zeros_like(gout) if h is None else h
    dph = gout * (1 - Z) * (1 - Ht * Ht)
    dpz = gout * (Hp - Ht) * Z * (1 - Z)
    dU2 = _adjoint(plan, n_ops, dph @ w[64:], C)
    dpr = dU2[:, cin:] * Hp * R * (1 - R) if h is not None else torch.zeros_like(dpz)
    dpzr = torch.cat([dpz, dpr], -1)
    dU1 = _adjoint(plan, n_ops, dpzr @ w[:64], C)
    dx = dU2[:, :cin] + dU1[:, :cin] if want_dx else None
    dh = gout * Z + dU2[:, cin:] * R + dU1[:, cin:] if want_dh else None
    return dph, dpzr, dx, dh


def fake_wgrad(n_ops, cin, S1, S2, dpzr, dph, has_bias):
    dw = torch.cat([(S1.t() @ dpzr).t(), (S2.t() @ dph).t()])
    return dw, (torch.cat([dpzr.sum(0), dph.sum(0)]) if has_bias else None)


@pytest.fixture()
def dense_rows(dense_graph_ops, monkeypatch):   # noqa: F811
    calls = []

    def counted(name, fn):
        def f(*a, **k):
            calls.append(name)
            return fn(*a, **k)
        return f
    monkeypatch.setattr(ops, "_require_cuda", lambda *a, **k: None)
    monkeypatch.setattr(ops, "gru_seq_supported", lambda *a, **k: False)        # the graph does not fit one SM
    monkeypatch.setattr(ops, "gru_rows_supported", lambda plan, n_ops, cin, cout: n_ops <= 1 and cin <= 16 and cout == 32)
    monkeypatch.setattr(ops, "gru_rows_pack_weights", counted("pack", fake_pack))
    monkeypatch.setattr(ops, "gru_rows_fwd", counted("fwd", fake_fwd))
    monkeypatch.setattr(ops, "gru_rows_bwd", counted("bwd", fake_bwd))
    monkeypatch.setattr(ops, "gru_rows_wgrad", counted("wgrad", fake_wgrad))
    return calls


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", CASES)
def test_wikimaths_host_logic_vs_reference_golden(golden_dir, dense_rows, case, fused):
    g = load(golden_dir)
    c = g["cases"][case]
    m = model_for(c, fused=fused)
    H0 = c["H0"].clone().requires_grad_(True) if "H0" in c else None
    out, losses = run(m, g, c, H0=H0)
    assert torch.allclose(out, c["out"], rtol=1e-4, atol=1e-5), float((out - c["out"]).abs().max())
    assert torch.allclose(losses, c["losses"], rtol=1e-4, atol=1e-6)
    for k, p in m.named_parameters():
        ref = c["grads"][k]
        assert p.grad is not None, k
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-6), k
    if H0 is not None:
        assert torch.allclose(H0.grad, c["gH0"], rtol=1e-3, atol=1e-3 * float(c["gH0"].abs().max()))
    S = g["X"].shape[0]
    if not fused:
        assert dense_rows == []
    elif H0 is None:                  # the parameters are fixed, so the pack runs once; one backward per snapshot
        assert dense_rows == ["pack"] + ["fwd", "bwd", "wgrad"] * S
    else:
        assert dense_rows == ["pack"] + ["fwd"] * S + ["bwd", "wgrad"] * S


def test_weight_pack_is_the_gate_weights_in_basis_order(dense_rows):
    torch.manual_seed(0)
    for K, cin, bias in ((2, 14, True), (1, 16, True), (2, 3, False)):
        m = GConvGRU(cin, 32, K, bias=bias)
        w, b = m._rows_packed()
        assert w.shape == (96, K * (cin + 32))
        for gi, g in enumerate("zrh"):
            assert torch.equal(w[32 * gi:32 * gi + 32], m._gate_weight(g).t())
            assert torch.equal(b[32 * gi:32 * gi + 32], m._gate_bias(g) if bias else torch.zeros(32))
        assert m._rows_packed()[0] is w                               # cached until a parameter changes
        with torch.no_grad():
            m.conv_x_z.lins[0].weight.add_(1.0)
        assert m._rows_packed()[0] is not w


def test_gradient_blocks_and_bias_copies_do_not_alias(golden_dir, dense_rows):
    """Every parameter receives exactly its block of the packed gradients; both ChebConvs of a gate receive the gate's bias gradient as
    separate tensors, and a second backward accumulates into each .grad on its own."""
    g = load(golden_dir)
    c = g["cases"]["K2_sym"]
    m = model_for(c)
    for _ in range(2):
        run(m, g, c)
    r = m.recurrent
    for gate in "zrh":
        bx, bh = getattr(r, f"conv_x_{gate}").bias, getattr(r, f"conv_h_{gate}").bias
        assert bx.grad.data_ptr() != bh.grad.data_ptr()
        assert torch.allclose(bx.grad, 2 * c["grads"][f"recurrent.conv_x_{gate}.bias"], rtol=1e-3, atol=1e-6)
        assert torch.allclose(bh.grad, bx.grad)
        for k in range(2):
            for side in "xh":
                key = f"recurrent.conv_{side}_{gate}.lins.{k}.weight"
                p = getattr(r, f"conv_{side}_{gate}").lins[k].weight
                assert p.grad.shape == p.shape
                assert torch.allclose(p.grad, 2 * c["grads"][key], rtol=1e-3, atol=2e-3 * float(c["grads"][key].abs().max()) + 1e-6), key


def test_routing(golden_dir, dense_rows, monkeypatch):
    g = load(golden_dir)
    ei, ew = g["edge_index"][:, :3000].long(), g["edge_weight"][:3000]
    N = 1068
    torch.manual_seed(1)
    X, H = torch.randn(N, 14), torch.randn(N, 32) * 0.5
    # outside the envelope: op-for-op, with gradients
    for m, x, h in ((GConvGRU(17, 32, 2), torch.randn(N, 17), H), (GConvGRU(14, 32, 3), X, H), (GConvGRU(14, 16, 2), X, H[:, :16]),
                    (GConvGRU(14, 32, 2), X.expand(2, N, 14), H.expand(2, N, 32))):
        m(x, ei, ew, h).sum().backward()
        assert all(p.grad is not None for p in m.parameters())
    assert dense_rows == []
    m = GConvGRU(14, 32, 2)
    m.fused_training = False                                          # training calls stay op-for-op ...
    m(X, ei, ew, H).sum().backward()
    assert dense_rows == []
    with torch.no_grad():                                             # ... inference does not depend on the switch
        m(X, ei, ew, H)
    assert dense_rows == ["pack", "fwd"]
    # X or H alone requiring grad takes the fused route, H = None has no state gradient
    m = GConvGRU(14, 32, 2).requires_grad_(False)
    ref = GConvGRU(14, 32, 2).requires_grad_(False)
    ref.load_state_dict(m.state_dict())
    ref.fused_training = False
    Xg, Hg = X.clone().requires_grad_(True), H.t().contiguous().t().requires_grad_(True)   # a non-contiguous H
    Xr, Hr = X.clone().requires_grad_(True), H.clone().requires_grad_(True)
    m(Xg, ei, ew, Hg).square().sum().backward()
    ref(Xr, ei, ew, Hr).square().sum().backward()
    assert torch.allclose(Xg.grad, Xr.grad, rtol=1e-4, atol=1e-5) and torch.allclose(Hg.grad, Hr.grad, rtol=1e-4, atol=1e-5)
    # a graph that fits one SM never consults the row-split entry
    dense_rows.clear()
    monkeypatch.setattr(ops, "gru_seq_supported", lambda *a, **k: True)
    monkeypatch.setattr(ops, "gru_rows_supported", lambda *a, **k: pytest.fail("row-split entry consulted"))
    m = GConvGRU(14, 32, 2)
    m(X, ei, ew, H).sum().backward()
    m(X, ei, ew).sum().backward()
    assert dense_rows == []
