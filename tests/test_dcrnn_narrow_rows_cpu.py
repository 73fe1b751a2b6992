"""Host side of BatchedDCRNN on the narrow row-split kernels (stmp_dcrnn_narrow_rows_*): the routing of a call (`BatchedDCRNN._rows_ok`),
the weight pack, the autograd Function `_DcrnnHoistedRowsFn` and the hand-off of its operands to `_weight_grads`, with every
library call replaced by a dense torch restatement of its contract on the dense DConv operators -- the output, gX and EVERY parameter
gradient against the unmodified reference (tests/golden/make_goldens_dcrnn_narrow_rows.py: BatchedDCRNN(2, 2, 3) on 2 000 nodes)."""
import gzip
import importlib.util
import os

import pytest
import torch

from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN
from pytorch_geometric_temporal_b200.nn.recurrent import dcrnn as dcrnn_mod
from test_dcrnn_rows_cpu import fake_rows_library
from test_modules_host_logic_cpu import dense_dconv_gcn_ops  # noqa: F401  (dense DConv operators + SpMM, one-SM kernels off)


def _load(golden_dir):
    with gzip.open(os.path.join(golden_dir, "dcrnn_narrow_rows_banded.pt.gz"), "rb") as f:
        g = torch.load(f, weights_only=False)
    spec = importlib.util.spec_from_file_location("_mk_nrows", os.path.join(golden_dir, "make_goldens_dcrnn_narrow_rows.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    g["edge_index"], g["edge_weight"], g["X"] = mod.inputs()
    return g


def _basis(plan, U, K):
    blocks, To, Ti = [U], None, None
    for k in range(1, K):
        if k == 1:
            To, Ti = plan.mats[0] @ U, plan.mats[1] @ U
        else:
            To, Ti = 2 * (plan.mats[0] @ To) - U, 2 * (plan.mats[1] @ Ti) - U
        blocks += [To, Ti]
    return torch.cat(blocks, -1)


def fake_pack(wz, wr, wh, cin, K):
    st = dcrnn_mod._stack_weight
    return st(wh).t().contiguous(), torch.cat([st(wz), st(wr)], dim=1).t().contiguous()


def _dense_forward(plan, x, wzrT, whsT, bz, br, bh, K, keep=None):
    B, T, N, cin = x.shape
    cout = whsT.size(0)
    H = x.new_zeros(B, N, cout)
    outs, stash, S1s, S2s = [], [], [], []
    for t in range(T):
        S1 = _basis(plan, torch.cat([x[:, t], H], -1), K)
        pzr = S1 @ wzrT.t() + (torch.cat([bz, br]) if bz is not None else 0.0)
        Z, R = torch.sigmoid(pzr[..., :cout]), torch.sigmoid(pzr[..., cout:])
        S2 = _basis(plan, torch.cat([x[:, t], H * R], -1), K)
        ph = S2 @ whsT.t() + (bh if bh is not None else 0.0)
        if keep is not None:
            pzr.retain_grad()
            ph.retain_grad()
            keep.append((pzr, ph))
        Ht = torch.tanh(ph)
        H = Z * H + (1 - Z) * Ht
        outs.append(H)
        stash.append(torch.cat([Z, R, Ht], -1))
        S1s.append(S1)
        S2s.append(S2)
    return torch.stack(outs, 1), stash, S1s, S2s


def fake_fwd(plan, x, wzrT, whsT, bz, br, bh, K, train=False):
    with torch.no_grad():
        out, stash, S1s, S2s = _dense_forward(plan, x, wzrT, whsT, bz, br, bh, K)
    if not train:
        return out
    B, T, N, _ = x.shape
    return out, torch.stack(stash), torch.cat(S1s).reshape(T * B, N, -1), torch.cat(S2s).reshape(T * B, N, -1)


def make_fake_bwd(state):
    def fake_bwd(plan, cin, K, gout, out, stash, wzrT, whsT, want_dx):
        """dph / dpzr as the gradients of the pre-activations, dX as X's: a dense autograd replay of the forward the fake kept"""
        x = state["x"].detach().clone().requires_grad_(True)
        keep = []
        with torch.enable_grad():
            bs = [None if v is None else v.detach() for v in state["b"]]          # the module's own biases: no gradient into them here
            o, *_ = _dense_forward(plan, x, wzrT, whsT, *bs, K, keep)
            (o * gout).sum().backward()
        dph = torch.stack([ph.grad for _, ph in keep])
        dpzr = torch.stack([pzr.grad for pzr, _ in keep])
        return dph, dpzr, x.grad if want_dx else None
    return fake_bwd


def fake_hoisted_rows(monkeypatch, served):
    """ops.dcrnn_hoisted_rows_fwd / _bwd replaced by the dense fakes, the library by `fake_rows_library(served)`; returns the call log"""
    calls, state = [], {}

    def fwd(plan, x, wzrT, whsT, bz, br, bh, K, win_start=None, horizon=None, train=False):
        assert win_start is None
        calls.append("fwd")
        state["x"], state["b"] = x, (bz, br, bh)
        return fake_fwd(plan, x, wzrT, whsT, bz, br, bh, K, train)

    def bwd(*a, **k):
        calls.append("bwd")
        return make_fake_bwd(state)(*a, **k)
    fake_rows_library(monkeypatch, served)
    monkeypatch.setattr(ops, "dcrnn_pack_bwd_weights", fake_pack)
    monkeypatch.setattr(ops, "dcrnn_hoisted_rows_fwd", fwd)
    monkeypatch.setattr(ops, "dcrnn_hoisted_rows_bwd", bwd)
    return calls


@pytest.fixture()
def dense_nrows(dense_dconv_gcn_ops, monkeypatch):   # noqa: F811
    return fake_hoisted_rows(monkeypatch, "stmp_dcrnn_narrow_rows_supported")


def _close(got, want, rtol=1e-4, atol=1e-5):
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _grad_close(got, ref):
    _close(got, ref, 1e-3, 1e-3 * max(ref.abs().max().item(), 1e-12))


def test_narrow_states_route_to_the_hoisted_rows_path_and_match_the_golden(golden_dir, dense_nrows):
    g = _load(golden_dir)
    m = BatchedDCRNN(2, 2, 3)
    m.load_state_dict(g["state"])
    ei, ew = g["edge_index"], g["edge_weight"]
    with torch.no_grad():
        out = m(g["X"], ei, ew)
    assert dense_nrows == ["fwd"]
    _close(out[:, g["out_steps"]], g["out"])
    X = g["X"].clone().requires_grad_(True)
    out = m(X, ei, ew)
    (out * torch.linspace(-1, 1, out.numel()).view_as(out)).sum().backward()
    assert dense_nrows == ["fwd", "fwd", "bwd"]
    _close(out[:, g["out_steps"]], g["out"])
    _grad_close(X.grad, g["gX"])
    for k, p in m.named_parameters():
        _grad_close(p.grad, g["grads"][k])


def test_narrow_fused_training_off_and_shapes_outside_the_envelope_keep_the_tiled_path(golden_dir, dense_nrows):
    g = _load(golden_dir)
    m = BatchedDCRNN(2, 2, 3)
    m.load_state_dict(g["state"])
    X = g["X"][:, :2]
    m._fused_training = False
    m(X.clone().requires_grad_(True), g["edge_index"], g["edge_weight"]).sum().backward()
    assert dense_nrows == []
    for cin, cout, K in ((2, 5, 3), (5, 2, 3), (2, 2, 5)):
        mm = BatchedDCRNN(cin, cout, K)
        with torch.no_grad():
            mm(torch.randn(1, 2, 2000, cin), g["edge_index"], g["edge_weight"])
    assert dense_nrows == []
