"""Host side of BatchedDCRNN on the row-split kernels (stmp_dcrnn_rows_*): the routing of a call (`BatchedDCRNN._rows_ok` and the envelope
of `ops.dcrnn_rows_supported`), the weight pack (`BatchedDCRNN._rows_packed`), the autograd Function `_DcrnnRowsFn` and the hand-off of the weight-gradient contraction to the
parameters, with every library call replaced by a dense torch restatement of its contract on the dense DConv operators -- the output, gX
and EVERY parameter gradient against the unmodified reference on the PEMS-BAY shape (tests/golden/make_goldens_dcrnn_rows.py; the output at steps 0, 1 and 11)."""
import gzip
import os

import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN, BatchedDCRNN
from pytorch_geometric_temporal_b200.nn.recurrent import dcrnn as dcrnn_mod
from test_modules_host_logic_cpu import _DensePair, dense_dconv_gcn_ops  # noqa: F401  (dense DConv operators + SpMM, one-SM kernels off)


def fake_rows_library(monkeypatch, served):
    """The library as the row-split routing sees it: the entry `served` (e.g. "stmp_dcrnn_rows_supported") admits every plan, and any other
    library call -- the other widths' entries included -- fails the test."""
    class Lib(object):
        def __getattr__(self, name):
            if name == served:
                return lambda handle, cin, cout, K: 1

            def refuse(*a):
                pytest.fail(f"{name} consulted")
            return refuse
    monkeypatch.setattr(_lib, "lib", Lib)
    monkeypatch.setattr(_DensePair, "handle", None, raising=False)


def _load(golden_dir):
    """the fixture of tests/golden/make_goldens_dcrnn_rows.py; `out` holds the steps `out_steps` of the output"""
    with gzip.open(os.path.join(golden_dir, "dcrnn_rows_pems_bay.pt.gz"), "rb") as f:
        g = torch.load(f, weights_only=False)
    g["edge_index"] = g["edge_index"].long()
    return g


def _basis(plan, U):
    return torch.cat([U, torch.matmul(plan.mats[0], U), torch.matmul(plan.mats[1], U)], dim=-1)


def _adjoint(plan, dS, C):
    return dS[..., :C] + torch.matmul(plan.mats[0].t(), dS[..., C:2 * C]) + torch.matmul(plan.mats[1].t(), dS[..., 2 * C:])


def fake_pack(wz, wr, wh, cin, K):
    st = dcrnn_mod._stack_weight
    return st(wh).t().contiguous(), torch.cat([st(wz), st(wr)], dim=1).t().contiguous()


def fake_fwd(plan, x, wzrT, whsT, bz, br, bh, win_start=None, horizon=None, train=False):
    if win_start is not None:
        x = torch.stack([x[s:s + horizon] for s in win_start.tolist()])
    B, T, N, cin = x.shape
    bzr = torch.cat([bz, br]) if bz is not None else 0.0
    bh = bh if bh is not None else 0.0
    ld = ops.dcrnn_bwd_basis_ld(cin, 32, 2)
    nb = 3 * (cin + 32)
    H = x.new_zeros(B, N, 32)
    outs, stash, S1s, S2s = [], [], [], []
    for t in range(T):
        S1 = _basis(plan, torch.cat([x[:, t], H], -1))
        pre = S1 @ wzrT.t() + bzr
        Z, R = torch.sigmoid(pre[..., :32]), torch.sigmoid(pre[..., 32:])
        S2 = _basis(plan, torch.cat([x[:, t], H * R], -1))
        Ht = torch.tanh(S2 @ whsT.t() + bh)
        H = Z * H + (1 - Z) * Ht
        outs.append(H)
        stash.append(torch.cat([Z, R, Ht], -1))
        S1s.append(torch.nn.functional.pad(S1, (0, ld - nb)))
        S2s.append(torch.nn.functional.pad(S2, (0, ld - nb)))
    out = torch.stack(outs, 1)
    if not train:
        return out
    return out, torch.stack(stash), torch.cat(S1s), torch.cat(S2s)


def fake_bwd(plan, cin, gout, out, stash, wzrT, whsT, want_dx):
    B, T, N, _ = gout.shape
    C = cin + 32
    dph_all, dpzr_all, dX = [None] * T, [None] * T, gout.new_zeros(B, T, N, cin)
    dH = gout.new_zeros(B, N, 32)
    for t in range(T - 1, -1, -1):
        Z, R, Ht = stash[t, ..., :32], stash[t, ..., 32:64], stash[t, ..., 64:]
        Hp = out[:, t - 1] if t else torch.zeros_like(Z)
        g = gout[:, t] + dH
        dph = g * (1 - Z) * (1 - Ht * Ht)
        dpz = g * (Hp - Ht) * Z * (1 - Z)
        dU2 = _adjoint(plan, dph @ whsT, C)
        dpr = dU2[..., cin:] * Hp * R * (1 - R)
        dpzr = torch.cat([dpz, dpr], -1)
        dU1 = _adjoint(plan, dpzr @ wzrT, C)
        dH = g * Z + dU2[..., cin:] * R + dU1[..., cin:]
        dX[:, t] = dU2[..., :cin] + dU1[..., :cin]
        dph_all[t], dpzr_all[t] = dph, dpzr
    return torch.stack(dph_all), torch.stack(dpzr_all), dX if want_dx else None


def fake_wgrad(cin, K, S1, S2, dpzr_all, dph_all, has_bias):
    C, nb = cin + 32, 3 * (cin + 32)
    S1, S2 = S1.reshape(-1, S1.size(-1))[:, :nb], S2.reshape(-1, S2.size(-1))[:, :nb]
    dpzr, dph = dpzr_all.reshape(-1, 64), dph_all.reshape(-1, 32)
    dWzr, dWh = S1.t() @ dpzr, S2.t() @ dph
    un = dcrnn_mod._unstack_weight_grad
    g = (un(dWzr[:, :32].contiguous(), K, C), un(dWzr[:, 32:].contiguous(), K, C), un(dWh, K, C))
    if not has_bias:
        return g + (None, None, None)
    return g + (dpzr[:, :32].sum(0), dpzr[:, 32:].sum(0), dph.sum(0))


@pytest.fixture()
def dense_rows(dense_dconv_gcn_ops, monkeypatch):   # noqa: F811
    calls = []

    def counted(name, fn):
        def f(*a, **k):
            calls.append(name)
            return fn(*a, **k)
        return f
    fake_rows_library(monkeypatch, "stmp_dcrnn_rows_supported")
    monkeypatch.setattr(ops, "dcrnn_pack_bwd_weights", counted("pack", fake_pack))
    monkeypatch.setattr(ops, "dcrnn_rows_fwd", counted("fwd", fake_fwd))
    monkeypatch.setattr(ops, "dcrnn_rows_bwd", counted("bwd", fake_bwd))
    monkeypatch.setattr(ops, "dcrnn_bwd_wgrad", counted("wgrad", fake_wgrad))
    return calls


def _model(g):
    m = BatchedDCRNN(2, 32, 2)
    m.load_state_dict(g["state"])
    return m


def _graph(n, e, seed):
    """random directed edges plus a ring, so every node has in- and out-degree >= 1 and DConv stays finite"""
    g = torch.Generator().manual_seed(seed)
    ring = torch.arange(n)
    pairs = torch.unique(torch.cat([torch.randint(0, n, (2, e), generator=g), torch.stack([ring, (ring + 1) % n])], 1), dim=1)
    return pairs[:, pairs[0] != pairs[1]]


def _grad_close(got, ref):
    assert torch.allclose(got, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-12)


@pytest.mark.parametrize("fused", [True, False])
def test_pems_bay_host_logic_vs_reference_golden(golden_dir, dense_rows, fused):
    g = _load(golden_dir)
    m = _model(g)
    m._fused_training = fused
    with torch.no_grad():
        out = m(g["X"], g["edge_index"], g["edge_weight"])
    assert torch.allclose(out[:, g["out_steps"]], g["out"], rtol=1e-4, atol=1e-5)
    assert dense_rows == ["pack", "fwd"]                       # inference is served by the row-split path whatever _fused_training says
    del dense_rows[:]
    X = g["X"].clone().requires_grad_(True)
    out = m(X, g["edge_index"], g["edge_weight"])
    (out * torch.linspace(-1, 1, out.numel()).view_as(out)).sum().backward()
    assert torch.allclose(out.detach()[:, g["out_steps"]], g["out"], rtol=1e-4, atol=1e-5)
    _grad_close(X.grad, g["gX"])
    for k, p in m.named_parameters():
        _grad_close(p.grad, g["grads"][k])
    assert dense_rows == (["fwd", "bwd", "wgrad"] if fused else [])   # the parameters did not change: the pack is reused


def test_no_input_gradient_and_no_bias(dense_rows):
    torch.manual_seed(0)
    ei = _graph(40, 160, 0)
    X = torch.randn(3, 4, 40, 3)
    for bias in (True, False):
        m = BatchedDCRNN(3, 32, 2, bias=bias)
        res = []
        for fused in (True, False):
            m._fused_training = fused
            m.zero_grad(set_to_none=True)
            out = m(X, ei, None)
            (out * out).sum().backward()
            res.append([out.detach()] + [p.grad.clone() for p in m.parameters()])
        for a, b in zip(*res):
            assert torch.allclose(a, b, rtol=1e-4, atol=1e-5 * float(b.abs().max()) + 1e-7)


def test_pack_is_the_stacked_weights_transposed_and_follows_parameter_updates(dense_rows):
    torch.manual_seed(1)
    m = BatchedDCRNN(4, 32, 2)
    whsT, wzrT = m._rows_packed()
    st = dcrnn_mod._stack_weight
    assert torch.equal(whsT, st(m.conv_x_h.weight).t()) and torch.equal(wzrT[:32], st(m.conv_x_z.weight).t())
    assert torch.equal(wzrT[32:], st(m.conv_x_r.weight).t()) and whsT.shape == (32, 108)
    assert m._rows_packed()[0] is whsT and dense_rows == ["pack"]
    with torch.no_grad():
        m.conv_x_h.weight.add_(1.0)
    assert torch.equal(m._rows_packed()[0], st(m.conv_x_h.weight).t()) and dense_rows == ["pack", "pack"]


def test_forward_indexed_reads_windows_in_place_without_gradients(dense_rows):
    torch.manual_seed(2)
    ei = _graph(30, 120, 2)
    series = torch.randn(50, 30, 2)
    starts = torch.tensor([0, 7, 31])
    m = BatchedDCRNN(2, 32, 2)
    with torch.no_grad():
        a = m.forward_indexed(series, starts, 12, ei, None)
        b = m(torch.stack([series[s:s + 12] for s in starts.tolist()]), ei, None)
    assert torch.equal(a, b)
    assert dense_rows == ["pack", "fwd", "fwd"]


def test_routing_outside_the_envelope(dense_rows):
    """cout 16, K = 3, cin 5 and the DCRNN cell stay on the tiled path; the envelope is checked in Python before any plan is consulted."""
    torch.manual_seed(3)
    ei = _graph(25, 90, 3)
    for cin, cout, K in ((2, 16, 2), (2, 32, 3), (5, 32, 2)):
        m = BatchedDCRNN(cin, cout, K)
        X = torch.randn(2, 3, 25, cin)
        with torch.no_grad():
            m(X, ei, None)
        m(X, ei, None).sum().backward()
    cell = DCRNN(2, 32, 2)
    cell(torch.randn(25, 2), ei, None).sum().backward()
    assert dense_rows == []


def test_envelope_is_checked_before_the_plan():
    """outside all three row-split envelopes the plan (None here) is never consulted"""
    for cin, cout, K in ((0, 32, 2), (5, 32, 2), (2, 16, 2), (2, 32, 1), (2, 32, 3), (2, 5, 3), (5, 2, 3), (2, 2, 5), (2, 0, 2),
                         (2, 2, 0), (2, 64, 1), (2, 64, 4), (5, 64, 2), (2, 16, 3)):
        assert ops.dcrnn_rows_supported(None, cin, cout, K) is False
