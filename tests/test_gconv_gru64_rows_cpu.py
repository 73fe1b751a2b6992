"""Host side of GConvGRU at 64 hidden channels on the 64-wide row-split cell kernels: the routing (`GConvGRU._rows_ok`), the weight pack
(`GConvGRU._rows_packed`), `ops._GruRowsFn` and the hand-off of the packed gradients (`GConvGRU._param_spec(rows=True)`), with every
library call replaced by a dense torch restatement of its contract (test_gconv_gru_rows_cpu.py's, at the width of its operands) on a dense
Chebyshev plan -- predictions, costs and every gradient against the unmodified reference (tests/golden/make_goldens_gconvgru64.py)."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU
from gconvgru64_seq import carried_h0, load, model_for, run_chickenpox, run_wikimaths
from gconvgru_seq import chickenpox_train_split
from test_modules_host_logic_cpu import dense_graph_ops  # noqa: F401  (dense Chebyshev plan + SpMM, one-SM inference off)
from wikimaths_seq import load as load_wikimaths


def _basis(plan, n_ops, U):
    return torch.cat([U] + [torch.matmul(plan.L, U)] * n_ops, dim=-1)


def _adjoint(plan, n_ops, dS, C):
    dU = dS[..., :C].clone()
    if n_ops:
        dU += torch.matmul(plan.L.t(), dS[..., C:2 * C])
    return dU


def fake_pack(n_ops, cin, wx, wh, bx=None, bh=None):
    Co = wh.size(-1)
    C = cin + Co
    w = wx.new_zeros(3 * Co, (n_ops + 1) * C)
    for g in range(3):
        for k in range(n_ops + 1):
            w[Co * g:Co * (g + 1), k * C:k * C + cin] = wx[g, k]
            w[Co * g:Co * (g + 1), k * C + cin:(k + 1) * C] = wh[g, k]
    return w, ((bx + bh).reshape(3 * Co) if bx is not None else wx.new_zeros(3 * Co))


def fake_fwd(plan, n_ops, x, h, w, b, train=False):
    Co = w.size(0) // 3
    H = x.new_zeros(x.size(0), Co) if h is None else h
    S1 = _basis(plan, n_ops, torch.cat([x, H], -1))
    pre = S1 @ w.t() + b
    Z, R = torch.sigmoid(pre[:, :Co]), torch.sigmoid(pre[:, Co:2 * Co])
    S2 = _basis(plan, n_ops, torch.cat([x, H * R], -1))
    Ht = torch.tanh((S2 @ w.t() + b)[:, 2 * Co:])
    out = Z * H + (1 - Z) * Ht
    return (out, torch.stack([Z, R, Ht]), S1, S2) if train else out


def fake_bwd(plan, n_ops, gout, h, stash, w, want_dx, want_dh, cin):
    Z, R, Ht = stash
    Co = gout.size(1)
    C = cin + Co
    Hp = torch.zeros_like(gout) if h is None else h
    dph = gout * (1 - Z) * (1 - Ht * Ht)
    dpz = gout * (Hp - Ht) * Z * (1 - Z)
    dU2 = _adjoint(plan, n_ops, dph @ w[2 * Co:], C)
    dpr = dU2[:, cin:] * Hp * R * (1 - R) if h is not None else torch.zeros_like(dpz)
    dpzr = torch.cat([dpz, dpr], -1)
    dU1 = _adjoint(plan, n_ops, dpzr @ w[:2 * Co], C)
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
    monkeypatch.setattr(ops, "gru_seq_supported", lambda *a, **k: False)
    monkeypatch.setattr(ops, "gru_rows_supported", lambda plan, n_ops, cin, cout: n_ops <= 1 and cin <= 16 and cout in (32, 64))
    monkeypatch.setattr(ops, "gru_rows_pack_weights", counted("pack", fake_pack))
    monkeypatch.setattr(ops, "gru_rows_fwd", counted("fwd", fake_fwd))
    monkeypatch.setattr(ops, "gru_rows_bwd", counted("bwd", fake_bwd))
    monkeypatch.setattr(ops, "gru_rows_wgrad", counted("wgrad", fake_wgrad))
    return calls


def _check(m, c, out, cost_or_losses, key):
    assert torch.allclose(out.double(), c["out"].double(), rtol=1e-4, atol=1e-5), float((out.double() - c["out"].double()).abs().max())
    assert torch.allclose(cost_or_losses.double(), c[key].double(), rtol=1e-4, atol=1e-6)
    for k, p in m.named_parameters():
        ref = c["grads"][k]
        assert p.grad is not None, k
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-6), k


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", ["K2_sym", "K1_sym", "K2_rw", "K2_sym_carried"])
def test_wikimaths_host_logic_vs_reference_golden(golden_dir, dense_rows, case, fused):
    g = load_wikimaths(golden_dir)
    c = load(golden_dir)["cases"][case]
    m = model_for(c, fused=fused)
    H0 = carried_h0(g["X"].size(1)).requires_grad_(True) if "gH0" in c else None
    out, losses = run_wikimaths(m, g["X"], g["Y"], g["edge_index"], g["edge_weight"], c["lambda_max"], H0)
    _check(m, c, out, losses, "losses")
    if H0 is not None:
        assert torch.allclose(H0.grad, c["gH0"], rtol=1e-3, atol=1e-3 * float(c["gH0"].abs().max()))
    S = g["X"].shape[0]
    if not fused:                     # training stays op-for-op
        assert dense_rows == []
    elif H0 is None:
        assert dense_rows == ["pack"] + ["fwd", "bwd", "wgrad"] * S
    else:
        assert dense_rows == ["pack"] + ["fwd"] * S + ["bwd", "wgrad"] * S


def test_chickenpox_host_logic_vs_reference_golden(golden_dir, dense_rows, monkeypatch):
    """20 nodes: at 64 channels the row-split route takes graphs that fit one SM as well (the one-SM kernel is never asked)."""
    monkeypatch.setattr(ops, "gru_seq_supported", lambda *a, **k: pytest.fail("one-SM entry consulted at 64 channels"))
    c = load(golden_dir)["cases"]["chickenpox"]
    ei, ew, X, Y = chickenpox_train_split()
    m = model_for(c, node_features=4)
    out, cost = run_chickenpox(m, X, Y, ei, ew)
    cost.backward()
    _check(m, c, out, cost.detach(), "cost")
    assert dense_rows == ["pack"] + ["fwd"] * X.size(0) + ["bwd", "wgrad"] * X.size(0)


def test_weight_pack_and_gradient_spec(dense_rows):
    torch.manual_seed(0)
    for K, cin, bias in ((2, 14, True), (1, 16, True), (2, 3, False)):
        m = GConvGRU(cin, 64, K, bias=bias)
        w, b = m._rows_packed()
        assert w.shape == (192, K * (cin + 64)) and b.shape == (192,)
        for gi, g in enumerate("zrh"):
            assert torch.equal(w[64 * gi:64 * gi + 64], m._gate_weight(g).t())
            assert torch.equal(b[64 * gi:64 * gi + 64], m._gate_bias(g) if bias else torch.zeros(64))
        spec, params = m._param_spec(rows=True)
        dw, db = torch.randn_like(w), torch.randn_like(b)
        for s, p, gr in zip(spec, params, ops._spec_grads(tuple(spec), dw, db)):      # every block is the parameter's own slice
            if s[0] == "w":
                _, r0, nr, c0, nc = s
                assert gr.shape == p.shape and torch.equal(gr, dw[r0:r0 + nr, c0:c0 + nc])
            else:
                assert gr.shape == p.shape and torch.equal(gr, db[s[1]:s[1] + s[2]])
        # the pack is the inverse of the spec: every parameter is found at its spec block
        for s, p in zip(spec, params):
            if s[0] == "w":
                _, r0, nr, c0, nc = s
                assert torch.equal(w[r0:r0 + nr, c0:c0 + nc], p.detach())


def test_routing(golden_dir, dense_rows, monkeypatch):
    g = load_wikimaths(golden_dir)
    ei, ew = g["edge_index"][:, :3000].long(), g["edge_weight"][:3000]
    N = 1068
    torch.manual_seed(1)
    X, H = torch.randn(N, 14), torch.randn(N, 64) * 0.5
    for m, x, h in ((GConvGRU(17, 64, 2), torch.randn(N, 17), H), (GConvGRU(14, 64, 3), X, H),
                    (GConvGRU(14, 64, 2), X.expand(2, N, 14), H.expand(2, N, 64))):
        m(x, ei, ew, h).sum().backward()
        assert all(p.grad is not None for p in m.parameters())
    assert dense_rows == []
    m = GConvGRU(14, 64, 2)
    m.fused_training = False
    m(X, ei, ew, H).sum().backward()
    assert dense_rows == []
    with torch.no_grad():
        m(X, ei, ew, H)
    assert dense_rows == ["pack", "fwd"]
    # at 32 channels a graph that fits one SM still never consults the row-split entry
    dense_rows.clear()
    monkeypatch.setattr(ops, "gru_seq_supported", lambda *a, **k: True)
    asked = []
    monkeypatch.setattr(ops, "gru_rows_supported", lambda plan, n_ops, cin, cout: asked.append(cout) or cout == 64)
    GConvGRU(14, 32, 2)(X, ei, ew, H[:, :32]).sum().backward()
    assert dense_rows == [] and asked == []
    GConvGRU(14, 64, 2)(X, ei, ew, H).sum().backward()                # ... and at 64 the row-split route is taken regardless
    assert dense_rows == ["pack", "fwd", "bwd", "wgrad"] and asked == [64]
