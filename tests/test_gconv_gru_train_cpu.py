"""Host side of GConvGRU training on the generic graph-GRU kernels (stmp_gru_seq_fwd with a stash + stmp_gru_bwd_*): the routing of a call
(`GConvGRU._train_ok`), the autograd Function `ops._GruSeqFn` and the hand-off of the prepacked-weight gradients (dwcat, dbcat) to the
module's parameters (`GConvGRU._param_spec`), with every library call replaced by a dense torch restatement of its contract -- outputs,
cost and EVERY gradient against the unmodified reference (tests/golden/make_goldens_gconvgru.py)."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU
from test_modules_host_logic_cpu import dense_graph_ops  # noqa: F401  (dense Chebyshev plan + SpMM, fused inference off)
from gconvgru_seq import load, model_for, run

GOLDENS = [f"gconvgru_chickenpox_K{K}_{n}" for K in (1, 2) for n in ("sym", "rw", "carried")] + ["gconvgru_metr_la_K2"]


def _wcol(m, cin, C):
    """wcat column of basis column m ([X | H] per block of the basis [U | Op0 U | ..])."""
    blk, c = divmod(m, C)
    return 96 + 4 * blk + c if c < cin else 32 * blk + c - cin


def _ops_of(plan, n_ops):
    return [plan.L] * n_ops            # the Chebyshev plan has one operator, the scaled Laplacian


def _basis(plan, n_ops, U):
    return torch.cat([U] + [torch.matmul(L, U) for L in _ops_of(plan, n_ops)], dim=-1)


def _A(plan, n_ops, X, Hp):
    """[Hp | Op0 Hp | Op1 Hp | X | Op0 X | Op1 X | 0] in wcat's column order."""
    A = X.new_zeros(*X.shape[:-1], 112)
    Ci = X.size(-1)
    A[..., 0:32], A[..., 96:96 + Ci] = Hp, X
    for k, L in enumerate(_ops_of(plan, n_ops)):
        A[..., 32 * (k + 1):32 * (k + 2)] = torch.matmul(L, Hp)
        A[..., 100 + 4 * k:100 + 4 * k + Ci] = torch.matmul(L, X)
    return A


def fake_seq_fwd(plan, n_ops, x, wcat, bcat, h0=None, h0_shared=False, wimage=None, stash=False):
    B, T, N, _ = x.shape
    H = x.new_zeros(B, N, 32) if h0 is None else h0.reshape(B, N, 32)
    out, st = x.new_empty(B, T, N, 32), x.new_empty(B, T, 3, N, 32)
    for t in range(T):
        pre = _A(plan, n_ops, x[:, t], H) @ wcat.t() + bcat
        Z, R = torch.sigmoid(pre[..., :32]), torch.sigmoid(pre[..., 32:64])
        Ht = torch.tanh((_A(plan, n_ops, x[:, t], H * R) @ wcat.t() + bcat)[..., 64:])
        H = Z * H + (1 - Z) * Ht
        out[:, t], st[:, t, 0], st[:, t, 1], st[:, t, 2] = H, Z, R, Ht
    return (out, st) if stash else out


def fake_pack_bwd_weights(n_ops, cin, wcat):
    C = cin + 32
    cols = [_wcol(m, cin, C) for m in range((n_ops + 1) * C)]
    return wcat[64:, cols].contiguous(), wcat[:64, cols].contiguous()


def fake_bwd_basis(plan, n_ops, x, out, h0, stash, S1, S2):
    B, T, N, Ci = x.shape
    w = (n_ops + 1) * (Ci + 32)
    for t in range(T):
        Hp = (x.new_zeros(B, N, 32) if h0 is None else h0) if t == 0 else out[:, t - 1]
        S1[t * B:(t + 1) * B, :, :w] = _basis(plan, n_ops, torch.cat([x[:, t], Hp], -1))
        S2[t * B:(t + 1) * B, :, :w] = _basis(plan, n_ops, torch.cat([x[:, t], Hp * stash[:, t, 1]], -1))


def _adjoint(plan, n_ops, dS, C):
    dU = dS[..., :C].clone()
    for k, L in enumerate(_ops_of(plan, n_ops)):
        dU += torch.matmul(L.t(), dS[..., (k + 1) * C:(k + 2) * C])
    return dU


def fake_bwd_seq(plan, n_ops, cin, gout, out, h0, stash, whsT, wzrT, dph_all, dpzr_all, dx, dh0):
    B, T, N, _ = gout.shape
    C = cin + 32
    carry = gout.new_zeros(B, N, 32)
    for t in range(T - 1, -1, -1):
        Z, R, Ht = stash[:, t, 0], stash[:, t, 1], stash[:, t, 2]
        Hp = (gout.new_zeros(B, N, 32) if h0 is None else h0) if t == 0 else out[:, t - 1]
        g = gout[:, t] + carry
        dph = g * (1 - Z) * (1 - Ht * Ht)
        dU2 = _adjoint(plan, n_ops, dph @ whsT, C)
        dpzr = torch.cat([g * (Hp - Ht) * Z * (1 - Z), dU2[..., cin:] * Hp * R * (1 - R)], -1)
        dU1 = _adjoint(plan, n_ops, dpzr @ wzrT, C)
        carry = g * Z + dU2[..., cin:] * R + dU1[..., cin:]
        dph_all[t], dpzr_all[t] = dph, dpzr
        if dx is not None:
            dx[:, t] = dU2[..., :cin] + dU1[..., :cin]
    dh0.copy_(carry)


def fake_bwd_wgrad(n_ops, cin, S1, S2, dpzr_all, dph_all, has_bias):
    C = cin + 32
    w = (n_ops + 1) * C
    s1, s2 = S1.reshape(-1, S1.size(-1))[:, :w], S2.reshape(-1, S2.size(-1))[:, :w]
    dzr, dh = dpzr_all.reshape(-1, 64), dph_all.reshape(-1, 32)
    dwcat = S1.new_zeros(96, 112)
    cols = [_wcol(m, cin, C) for m in range(w)]
    dwcat[:64, cols] = (s1.t() @ dzr).t()
    dwcat[64:, cols] = (s2.t() @ dh).t()
    return dwcat, (torch.cat([dzr.sum(0), dh.sum(0)]) if has_bias else None)


@pytest.fixture()
def dense_kernels(dense_graph_ops, monkeypatch):   # noqa: F811
    calls = []

    def counted(name, fn):
        def f(*a, **k):
            calls.append(name)
            return fn(*a, **k)
        return f
    monkeypatch.setattr(ops, "_require_cuda", lambda *a, **k: None)
    monkeypatch.setattr(ops, "gru_seq_supported", lambda *a, **k: True)
    monkeypatch.setattr(ops, "gru_bwd_supported", lambda *a, **k: True)
    monkeypatch.setattr(ops, "gru_weight_image", lambda W, b: None)
    monkeypatch.setattr(ops, "gru_seq_fwd", counted("fwd", fake_seq_fwd))
    monkeypatch.setattr(ops, "gru_pack_bwd_weights", fake_pack_bwd_weights)
    monkeypatch.setattr(ops, "gru_bwd_basis", fake_bwd_basis)
    monkeypatch.setattr(ops, "gru_bwd_seq", counted("bwd", fake_bwd_seq))
    monkeypatch.setattr(ops, "gru_bwd_wgrad", fake_bwd_wgrad)
    return calls


def _check(m, g, out, loss, H0):
    assert torch.allclose(out, g["out"], rtol=1e-4, atol=1e-5), float((out - g["out"]).abs().max())
    assert torch.allclose(loss, g["loss"], rtol=1e-4, atol=1e-6)
    for k, p in m.named_parameters():
        ref = g["grads"][k]
        assert p.grad is not None, k
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-6), k
    if H0 is not None:
        assert torch.allclose(H0.grad, g["gH0"], rtol=1e-3, atol=1e-3 * float(g["gH0"].abs().max()))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", GOLDENS)
def test_gconvgru_training_host_logic_vs_reference_golden(golden_dir, dense_kernels, name, fused):
    g = load(golden_dir, name)
    m = model_for(g, fused=fused)
    H0 = g["H0"].clone().requires_grad_(True) if "H0" in g else None
    out, loss = run(m, g, H0=H0)
    loss.backward()
    _check(m, g, out, loss, H0)
    steps = g["X"].shape[0]
    assert dense_kernels == (["fwd"] * steps + ["bwd"] * steps if fused else [])


def test_bias_gradients_do_not_alias(golden_dir, dense_kernels):
    """Both ChebConvs of a gate receive the gate's bias gradient; a second backward accumulates into each .grad separately."""
    g = load(golden_dir, "gconvgru_chickenpox_K2_sym")
    m = model_for(g)
    for _ in range(2):
        run(m, g)[1].backward()
    r = m.recurrent
    for gate in "zrh":
        bx, bh = getattr(r, f"conv_x_{gate}").bias, getattr(r, f"conv_h_{gate}").bias
        assert bx.grad.data_ptr() != bh.grad.data_ptr()
        assert torch.allclose(bx.grad, 2 * g["grads"][f"recurrent.conv_x_{gate}.bias"], rtol=1e-3, atol=1e-6)
        assert torch.allclose(bh.grad, bx.grad)


def test_routing(golden_dir, dense_kernels):
    """Outside the envelope (K = 3, out_channels != 32, in_channels > 4, 3-D X, fused_training = False) the op-for-op path runs, and
    still produces its gradients; X or H alone requiring grad takes the fused route."""
    g = load(golden_dir, "gconvgru_chickenpox_K2_sym")
    ei, ew = g["edge_index"], g["edge_weight"]
    torch.manual_seed(0)
    X, H = torch.randn(20, 4), torch.randn(20, 32) * 0.5
    for m, x, h in ((GConvGRU(4, 32, 3), X, H), (GConvGRU(4, 16, 2), X, H[:, :16]), (GConvGRU(5, 32, 2), torch.randn(20, 5), H),
                    (GConvGRU(4, 32, 2), X.expand(3, 20, 4), H.expand(3, 20, 32))):
        m(x, ei, ew, h).sum().backward()
        assert all(p.grad is not None for p in m.parameters())
    m = GConvGRU(4, 32, 2)
    m.fused_training = False
    m(X, ei, ew, H).sum().backward()
    assert dense_kernels == []
    m = GConvGRU(4, 32, 2).requires_grad_(False)
    Xg, Hg = X.clone().requires_grad_(True), H.t().contiguous().t().requires_grad_(True)       # a non-contiguous H
    ref = GConvGRU(4, 32, 2).requires_grad_(False)
    ref.load_state_dict(m.state_dict())
    ref.fused_training = False
    Xr, Hr = X.clone().requires_grad_(True), H.clone().requires_grad_(True)
    m(Xg, ei, ew, Hg).square().sum().backward()
    ref(Xr, ei, ew, Hr).square().sum().backward()
    assert dense_kernels == ["fwd", "bwd"]
    assert torch.allclose(Xg.grad, Xr.grad, rtol=1e-4, atol=1e-5) and torch.allclose(Hg.grad, Hr.grad, rtol=1e-4, atol=1e-5)
