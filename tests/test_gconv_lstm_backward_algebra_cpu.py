"""Host-side algebra of the hand-written GConvLSTM cell backward (`nn/recurrent/gconv_lstm.py::_LstmCellFn`) checked on the CPU
against autograd through the op-for-op path and against the reference module's gradients: the CUDA entry points are replaced by
dense torch stand-ins that follow the contracts of include/stmp.h (stmp_spmm on column blocks, stmp_gemm_lstm_f32, stmp_gemm_f32
with a strided `out`, stmp_lstm_gate_bwd).  Pins, without a GPU: the recompute-in-backward scheme, the gate derivatives' call
shapes, dS = dpre W^T in two column halves, the in-place adjoint of the Chebyshev recurrence, the chunked weight gradient, the
peephole / bias reductions and the reuse of one (W, bias) graph across the steps of a sequence."""
import pytest
import torch

import pytorch_geometric_temporal_b200.nn.recurrent._cheb as cheb_mod
import pytorch_geometric_temporal_b200.nn.recurrent.gconv_lstm as L
from oracle import pyg, recurrent as R
from pytorch_geometric_temporal_b200 import ops


class _Plan(object):
    def __init__(self, Lm):
        self.L = Lm


def _install(monkeypatch):
    def spmm_cols(plan, op, buf, src, dst, width, alpha=1.0, z_col=None, beta=0.0, transposed=False):
        A = plan.L.t() if transposed else plan.L
        y = alpha * torch.matmul(A, buf[..., src:src + width])
        if z_col is not None:
            y = y + beta * buf[..., z_col:z_col + width]
        buf[..., dst:dst + width] = y

    def spmm(plan, op, x, alpha=1.0, z=None, beta=0.0, att=None):
        y = alpha * torch.matmul(plan.L, x)
        return y if z is None else y + beta * z

    def gemm_prepack(W):
        return W.clone()                                  # "packed" = the fp32 matrix itself

    def vectors(n, *vs):                                  # per-channel operands: exactly n elements, or absent where the ABI allows it
        assert all(v is None or v.numel() == n for v in vs), [None if v is None else v.numel() for v in vs]

    def gemm(A, packed, K, N, bias=None, out=None):
        assert A.numel() % K == 0                         # the kernel walks M = A.numel() / K rows
        vectors(N, bias)
        C = A.reshape(-1, K) @ packed
        if bias is not None:
            C = C + bias
        if out is not None:
            out.copy_(C)
            return out
        return C.reshape(*A.shape[:-1], N)

    def gemm_lstm(A, packed, K, cout, cb, cell, wci, wcf, wco, bi, bf, bc, bo):
        # stmp_gemm_lstm_f32 reads one cell row and writes one H' / C' row per row of A: M = A.numel() / K of each
        assert A.numel() % K == 0 and cell.numel() == (A.numel() // K) * cout, (tuple(A.shape), K, tuple(cell.shape))
        vectors(4 * cout, cb)
        vectors(cout, wci, wcf, wco, bi, bf, bc, bo)
        pre = A @ packed + (0 if cb is None else cb)
        pi, pf, pc, po = (pre[..., j * cout:(j + 1) * cout] for j in range(4))
        I, Fg = torch.sigmoid(pi + wci * cell + bi), torch.sigmoid(pf + wcf * cell + bf)
        Cn = Fg * cell + I * torch.tanh(pc + bc)
        return torch.sigmoid(po + wco * Cn + bo) * torch.tanh(Cn), Cn

    def lstm_gate_bwd(pre, c_old, c_new, gh, gc, wci, wcf, wco, bi, bf, bc, bo):
        Co = c_old.size(-1)
        rows = c_old.numel() // Co                        # stmp_lstm_gate_bwd walks rows x Co elements of every operand
        assert pre.numel() == rows * 4 * Co and all(t is None or t.numel() == rows * Co for t in (c_new, gh, gc))
        vectors(Co, wci, wcf, wco, bi, bf, bc, bo)
        pi, pf, pc, po = (pre[:, j * Co:(j + 1) * Co] for j in range(4))
        iv, fv = torch.sigmoid(pi + wci * c_old + bi), torch.sigmoid(pf + wcf * c_old + bf)
        tv, ov, tc = torch.tanh(pc + bc), torch.sigmoid(po + wco * c_new + bo), torch.tanh(c_new)
        g = torch.zeros_like(c_old) if gh is None else gh
        dpo = g * tc * ov * (1 - ov)
        dcn = (0 if gc is None else gc) + g * ov * (1 - tc * tc) + dpo * wco
        dpi, dpf, dpc = dcn * tv * iv * (1 - iv), dcn * c_old * fv * (1 - fv), dcn * iv * (1 - tv * tv)
        return torch.cat([dpi, dpf, dpc, dpo], dim=1), dcn * fv + dpi * wci + dpf * wcf

    for name, fn in dict(spmm_cols=spmm_cols, spmm=spmm, gemm_prepack=gemm_prepack, gemm=gemm, gemm_lstm=gemm_lstm,
                         lstm_gate_bwd=lstm_gate_bwd).items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(L, "_require_cuda", lambda *a, **k: None)

    def plan(self, edge_index, edge_weight, num_nodes, normalization, lambda_max, batch=None):
        e, w = pyg.cheb_norm(edge_index, num_nodes, edge_weight, normalization, self._lambda_value(lambda_max))
        M = torch.zeros(num_nodes, num_nodes)
        M.index_put_((e[1], e[0]), w, accumulate=True)
        return _Plan(M)
    monkeypatch.setattr(cheb_mod.ChebPlanMixin, "_cheb_plan", plan)


@pytest.mark.parametrize("K,batched", [(3, False), (2, True), (1, False)])
def test_lstm_cell_backward_matches_autograd_and_reference(monkeypatch, K, batched):
    _install(monkeypatch)
    torch.manual_seed(K)
    n, Ci, Co, T = 24, 32, 32, 3
    ei = torch.stack([torch.randint(0, n, (90,)), torch.randint(0, n, (90,))])
    ei = torch.unique(ei[:, ei[0] != ei[1]], dim=1)
    ew = torch.rand(ei.size(1)) + 0.1
    lead = (2, n) if batched else (n,)
    X = (torch.randn(T, *lead, Ci) * 0.5)
    a, b = L.GConvLSTM(Ci, Co, K), L.GConvLSTM(Ci, Co, K)
    for p in a.parameters():                      # zero biases would hide bias-gradient mistakes
        if p.dim() == 1 or p.size(0) == 1:
            torch.nn.init.normal_(p, std=0.2)
    b.load_state_dict(a.state_dict())
    b.fused_training = False
    outs = {}
    for name, m in (("fused", a), ("autograd", b)):
        x = X.clone().requires_grad_(True)
        H = C = None
        loss = 0
        for t in range(T):
            H, C = m(x[t], ei, ew, H, C)
            loss = loss + (H * torch.linspace(-1, 1, H.numel()).view_as(H)).sum() + 0.3 * C.square().sum()
        loss.backward()
        outs[name] = (H.detach(), C.detach(), x.grad, {k: p.grad.clone() for k, p in m.named_parameters()})
    assert a._train_cache is None                                   # the shared (W, bias) graph was dropped by the backward pass
    fH, fC, fx, fp = outs["fused"]
    aH, aC, ax, ap = outs["autograd"]
    assert torch.allclose(fH, aH, rtol=1e-5, atol=1e-6) and torch.allclose(fC, aC, rtol=1e-5, atol=1e-6)
    assert torch.allclose(fx, ax, rtol=1e-4, atol=1e-5), float((fx - ax).abs().max())
    for k in ap:
        assert torch.allclose(fp[k], ap[k], rtol=1e-4, atol=1e-4 * float(ap[k].abs().max()) + 1e-6), (k, float((fp[k] - ap[k]).abs().max()))
    if not batched:
        # and the reference's own cell (oracle restatement, pinned bit-exactly to the unmodified module) gives the same gradients
        p = {k: v.detach().clone().requires_grad_(True) for k, v in a.state_dict().items()}
        x = X.clone().requires_grad_(True)
        H = C = None
        loss = 0
        for t in range(T):
            H, C = R.gconv_lstm_cell(p, x[t], ei, ew, H, C)
            loss = loss + (H * torch.linspace(-1, 1, H.numel()).view_as(H)).sum() + 0.3 * C.square().sum()
        loss.backward()
        assert torch.allclose(fx, x.grad, rtol=1e-4, atol=1e-5)
        for k in fp:
            assert torch.allclose(fp[k], p[k].grad, rtol=1e-4, atol=1e-4 * float(p[k].grad.abs().max()) + 1e-6), k


@pytest.mark.parametrize("train", [True, False])
def test_state_shared_across_a_batch_matches_reference(monkeypatch, train):
    """X (B, N, F) with H, C (N, out): the reference sums conv(X), conv(H) and w_c * C elementwise, so one state serves every window
    and dH / dC sum over the batch.  Training runs `_LstmCellFn`, a `no_grad` call the fused GEMM + gate epilogue; both must hand the
    kernels a state row for every row of the basis."""
    _install(monkeypatch)
    calls = []
    gemm_lstm = ops.gemm_lstm
    monkeypatch.setattr(ops, "gemm_lstm", lambda *a: calls.append(tuple(a[0].shape)) or gemm_lstm(*a))
    torch.manual_seed(5)
    n, Ci, Co, K, B = 24, 32, 32, 3, 3
    ei = torch.stack([torch.randint(0, n, (90,)), torch.randint(0, n, (90,))])
    ei = torch.unique(ei[:, ei[0] != ei[1]], dim=1)
    ew = torch.rand(ei.size(1)) + 0.1
    m = L.GConvLSTM(Ci, Co, K)
    for p in m.parameters():
        if p.dim() == 1 or p.size(0) == 1:
            torch.nn.init.normal_(p, std=0.2)
    X, H0, C0 = torch.randn(B, n, Ci) * 0.5, torch.randn(n, Co) * 0.5, torch.randn(n, Co) * 0.5
    wh, wc = torch.randn(B, n, Co), torch.randn(B, n, Co)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    leaves = [t.clone().requires_grad_(True) for t in (X, H0, C0)]
    rh, rc = R.gconv_lstm_cell(p, *leaves[:1], ei, ew, *leaves[1:])
    assert rh.shape == (B, n, Co)
    ((rh * wh).sum() + (rc * wc).sum()).backward()
    got = [t.clone().requires_grad_(train) for t in (X, H0, C0)]
    with torch.set_grad_enabled(train):
        h, c = m(got[0], ei, ew, got[1], got[2])
    assert calls == [(B, n, K * (Ci + Co))], calls                    # one fused GEMM over all B N rows, not the autograd path
    assert torch.allclose(h, rh, rtol=1e-5, atol=1e-6) and torch.allclose(c, rc, rtol=1e-5, atol=1e-6)
    if not train:
        return
    ((h * wh).sum() + (c * wc).sum()).backward()
    for name, a, b in zip(("dX", "dH", "dC"), got, leaves):
        assert a.grad.shape == b.grad.shape and torch.allclose(a.grad, b.grad, rtol=1e-4, atol=1e-5), (name, float((a.grad - b.grad).abs().max()))
    for k, q in m.named_parameters():
        assert torch.allclose(q.grad, p[k].grad, rtol=1e-4, atol=1e-4 * float(p[k].grad.abs().max()) + 1e-6), k
