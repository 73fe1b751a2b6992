"""Host side of TGCN training with a carried state (stmp_tgcn_attn_fwd + stmp_tgcn_cell_bwd): the routing of each step, the
differentiable folding `TGCN._fold3` and the chaining of the steps through autograd, with the kernel pairs replaced by dense
differentiable restatements of their arithmetic -- outputs, loss and EVERY gradient against the unmodified reference
(tests/golden/make_goldens_tgcn.py)."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import TGCN, TGCN2
from test_modules_host_logic_cpu import dense_dconv_gcn_ops  # noqa: F401  (dense GCN plan + SpMM, no fused inference kernels)
from tgcn_seq import load, model_for, run


def _gates(L, x, h, A, Bm, c):
    ax = torch.matmul(L, x[..., 0])                                             # A^X, one period
    pre = lambda g, Hp: ax @ A[:, 32 * g:32 * g + 32] + Hp @ Bm[:, 32 * g:32 * g + 32] + c[32 * g:32 * g + 32]
    Z, R = torch.sigmoid(pre(0, h)), torch.sigmoid(pre(1, h))
    return Z * h + (1 - Z) * torch.tanh(pre(2, h * R))


@pytest.fixture()
def dense_kernels(dense_dconv_gcn_ops, monkeypatch):   # noqa: F811
    calls = []

    def fake_attn_train(plan, x, A, Bm, c, probs=None):
        calls.append(("attn", tuple(x.shape)))
        return _gates(plan.mats[0], x, torch.zeros(*x.shape[:2], 32), A, Bm, c)

    def fake_cell_train(plan, x, h, A, Bm, c):
        calls.append(("cell", tuple(x.shape), tuple(h.shape)))
        return _gates(plan.mats[0], x, h, A, Bm, c)
    monkeypatch.setattr(ops, "tgcn_attn_train", fake_attn_train)
    monkeypatch.setattr(ops, "tgcn_cell_train", fake_cell_train)
    return calls


def _check(m, g, out, loss):
    assert torch.allclose(out, g["out"], rtol=1e-4, atol=1e-5), float((out - g["out"]).abs().max())
    assert torch.allclose(loss, g["loss"], rtol=1e-4, atol=1e-6)
    for k, p in m.named_parameters():
        ref = g["grads"][k]
        assert p.grad is not None, k
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-6), k


@pytest.mark.parametrize("name,B,N", [("tgcn2_seq_metr_la_grads", 8, 207), ("tgcn2_seq_pems_bay_grads", 4, 325)])
def test_batched_tgcn_loop_host_logic_vs_reference_golden(golden_dir, dense_kernels, name, B, N):
    g = load(golden_dir, name)
    m = model_for(g)
    out, loss = run(m, g)
    loss.backward()
    _check(m, g, out, loss)
    # step 0 (H = None) trains on the H = None kernel pair, the 11 steps with a carried state on the cell backward
    assert dense_kernels == [("attn", (B, N, 2, 1))] + [("cell", (B, N, 2, 1), (B, N, 32))] * 11


def test_tgcn_chickenpox_loop_host_logic_vs_reference_golden(golden_dir, dense_kernels):
    g = load(golden_dir, "tgcn_chickenpox_seq_grads")
    m = model_for(g)
    H0 = g["H0"].clone().requires_grad_(True)
    out, loss = run(m, g, H0=H0)
    loss.backward()
    _check(m, g, out, loss)
    assert torch.allclose(H0.grad, g["gH0"], rtol=1e-3, atol=1e-3 * float(g["gH0"].abs().max()))
    assert dense_kernels == [("cell", (1, 20, 4, 1), (1, 20, 32))] * 24


def test_carried_state_routing(golden_dir, dense_kernels):
    """Only a call the cell backward serves takes it: an input gradient, out_channels != 32, in_channels > 4, fused_training = False or
    a state of another shape stay on the op-for-op path (and still produce their gradients)."""
    g = load(golden_dir, "tgcn2_seq_metr_la_grads")
    ei, ew = g["edge_index"], g["edge_weight"]
    torch.manual_seed(0)
    X, H = torch.randn(2, 207, 2), torch.randn(2, 207, 32) * 0.5
    Xg = X.clone().requires_grad_(True)
    TGCN2(2, 32, 2)(Xg, ei, ew, H).sum().backward()
    assert Xg.grad is not None
    TGCN2(2, 16, 2)(X, ei, ew, H[..., :16]).sum().backward()
    TGCN2(5, 32, 2)(torch.randn(2, 207, 5), ei, ew, H).sum().backward()
    m = TGCN2(2, 32, 2)
    m.fused_training = False
    m(X, ei, ew, H).sum().backward()
    TGCN(2, 32)(X[0], ei, ew, H[:1]).sum().backward()                           # (1, N, 32) state for an (N, F) input
    assert dense_kernels == []
    Hl = H.clone().requires_grad_(True)
    TGCN2(2, 32, 2)(X, ei, ew, Hl).sum().backward()
    TGCN(2, 32)(X[0], ei, ew, H[0]).sum().backward()
    assert Hl.grad is not None
    assert dense_kernels == [("cell", (2, 207, 2, 1), (2, 207, 32)), ("cell", (1, 207, 2, 1), (1, 207, 32))]
