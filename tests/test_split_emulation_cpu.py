"""The fp16 hi/lo operand split of the wgmma GEMMs (k_gemm_split: hi = fp16(v), lo = fp16(v - hi), products lo*hi + hi*lo + hi*hi)
emulated bit for bit on the CPU, and the hand-written GConvLSTM cell backward (`nn/recurrent/gconv_lstm.py::_LstmCellFn`) run with
that emulation in place of `ops.gemm` at the gradient scale a mean loss produces.

The split carries 22 mantissa bits only while both halves are normal fp16 numbers (|v| between about 2^-3 and 2^15); below 3e-8 both
halves round to zero.  Gradients of a masked-MAE mean loss are 1e-6 .. 1e-10, so `dpre @ W^T` must see dpre prescaled into range
(`_split_prescale`), otherwise backpropagation through time is cut off after the last step.  The kernels other than the GEMMs are
dense torch stand-ins following include/stmp.h, as in test_gconv_lstm_backward_algebra_cpu.py."""
import pytest
import torch

import pytorch_geometric_temporal_b200.nn.recurrent._cheb as cheb_mod
import pytorch_geometric_temporal_b200.nn.recurrent.gconv_lstm as L
from oracle import pyg, recurrent as R
from pytorch_geometric_temporal_b200 import distributed as D, ops


def _split(v: torch.Tensor):
    """fp16 (hi, lo) of an fp32 tensor as __float2half_rn rounds it (nearest even, subnormals kept, overflow to inf)."""
    hi = v.half()
    return hi, (v - hi.float()).half()


def split_matmul(A: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """A @ W as the wgmma kernels compute it.  Each fp16 x fp16 product is exact in fp32; the three passes are summed in float64
    here (fp32 accumulators on the device), so this isolates the error of the operand split itself."""
    Ah, Al = (t.double() for t in _split(A))
    Wh, Wl = (t.double() for t in _split(W))
    return (Al @ Wh + Ah @ Wl + Ah @ Wh).float()


def test_split_emulation_error_floor():
    """The emulation shows the split's contract: relative 2^-22 per product inside the normal band, an absolute floor of about
    2^-25 per operand element below it, and all bits lost under 3e-8."""
    g = torch.Generator().manual_seed(0)
    A = torch.randn(64, 96, generator=g)
    W = torch.randn(96, 32, generator=g) * 0.1
    for scale in (1.0, 1e-4, 1e-6, 1e-8):
        As = A * scale
        ref = As.double() @ W.double()
        err = (split_matmul(As, W).double() - ref).abs()
        bound = 2.0 ** -22 * (As.double().abs() @ W.double().abs()) + 2.0 ** -25 * (As.double().abs().sum(1, keepdim=True) + W.double().abs().sum(0))
        assert bool((err <= 2 * bound).all()), (scale, float((err / bound).max()))
        rel = float(err.max() / ref.abs().max())
        if scale == 1.0:
            assert rel < 1e-6, rel
        if scale == 1e-8:
            assert rel > 0.5, rel                     # hi and lo both flush to zero: the product is gone
    # an exact power-of-two prescale into the normal band restores the full accuracy, and undoing it is exact
    As = A * 1e-8
    s = 2.0 ** 40
    ref = As.double() @ W.double()
    err = (split_matmul(As * s, W) / s).double() - ref
    assert float(err.abs().max() / ref.abs().max()) < 1e-6


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
        return W.detach().clone()                         # "packed" = the fp32 matrix; the split happens in split_matmul

    def gemm(A, packed, K, N, bias=None, out=None):
        C = split_matmul(A.reshape(-1, K), packed)
        if bias is not None:
            C = C + bias
        if out is not None:
            out.copy_(C)
            return out
        return C.reshape(*A.shape[:-1], N)

    def gemm_lstm(A, packed, K, cout, cb, cell, wci, wcf, wco, bi, bf, bc, bo):
        pre = split_matmul(A.reshape(-1, K), packed).reshape(*A.shape[:-1], 4 * cout) + (0 if cb is None else cb)
        pi, pf, pc, po = (pre[..., j * cout:(j + 1) * cout] for j in range(4))
        I, Fg = torch.sigmoid(pi + wci * cell + bi), torch.sigmoid(pf + wcf * cell + bf)
        Cn = Fg * cell + I * torch.tanh(pc + bc)
        return torch.sigmoid(po + wco * Cn + bo) * torch.tanh(Cn), Cn

    def lstm_gate_bwd(pre, c_old, c_new, gh, gc, wci, wcf, wco, bi, bf, bc, bo):
        Co = c_old.size(-1)
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


def _run(cell, head, X, Y, ei, ew):
    x = X.clone().requires_grad_(True)
    H = C = None
    for t in range(X.size(0)):
        H, C = cell(x[t], ei, ew, H, C)
    D.masked_mae_loss(head(H), Y).backward()
    grads = {k: p.grad.clone() for k, p in list(cell.named_parameters()) + [("head." + k, p) for k, p in head.named_parameters()]}
    grads["X"] = x.grad
    for p in list(cell.parameters()) + list(head.parameters()):
        p.grad = None
    return grads


def _oracle(cell, head, X, Y, ei, ew):
    """The same loss in float64 autograd through the reference cell (oracle restatement of gconv_lstm.py:204-238)."""
    p = {k: v.detach().double().requires_grad_(True) for k, v in cell.state_dict().items()}
    hw, hb = (t.detach().double().requires_grad_(True) for t in (head.weight, head.bias))
    x = X.double().requires_grad_(True)
    H = torch.zeros(*X.shape[1:-1], cell.out_channels, dtype=torch.float64)
    C = torch.zeros_like(H)
    for t in range(X.size(0)):
        H, C = R.gconv_lstm_cell(p, x[t], ei, ew.double(), H, C)
    D.masked_mae_loss_reference(torch.nn.functional.linear(H, hw, hb), Y.double()).backward()
    grads = {k: v.grad for k, v in p.items()}
    grads["head.weight"], grads["head.bias"], grads["X"] = hw.grad, hb.grad, x.grad
    return grads


def test_lstm_cell_backward_at_mean_loss_scale(monkeypatch):
    """cfg5's cell, GConvLSTM(64, 64, K=3) under a Linear head and masked MAE, over 12 steps.  The fused backward with the emulated
    split must be as close to float64 as the op-for-op fp32 path is: at most 4x its error plus 1e-6 of the gradient's scale."""
    _install(monkeypatch)
    torch.manual_seed(0)
    n, B, T, Fd = 160, 4, 12, 64
    ei = torch.stack([torch.randint(0, n, (800,)), torch.randint(0, n, (800,))])
    ei = torch.unique(ei[:, ei[0] != ei[1]], dim=1)
    ew = torch.rand(ei.size(1)) + 0.1
    X = torch.randn(T, B, n, Fd)
    Y = torch.randn(B, n, Fd)
    Y[Y.abs() < 0.3] = 0                                              # masked targets, as in the traffic datasets
    cell, head = L.GConvLSTM(Fd, Fd, 3), torch.nn.Linear(Fd, Fd)
    for pr in cell.parameters():                                      # non-zero biases and peepholes
        if pr.dim() == 1 or pr.size(0) == 1:
            torch.nn.init.normal_(pr, std=0.2)
    fused = _run(cell, head, X, Y, ei, ew)
    cell.fused_training = False
    plain = _run(cell, head, X, Y, ei, ew)
    ref = _oracle(cell, head, X, Y, ei, ew)
    assert float(ref["X"][0].abs().max()) < 1e-6                      # the first step's gradients are deep in the range the split loses
    for g in (fused, plain, ref):                                     # dX per step: the early steps are the ones a range loss cuts off
        g.update({f"X[{t}]": xt for t, xt in enumerate(g.pop("X"))})
    for k, r in ref.items():
        err = float((fused[k].double() - r).abs().max())
        base = float((plain[k].double() - r).abs().max())
        scale = float(r.abs().max())
        assert err <= 4 * base + 1e-6 * scale, (k, err, base, scale)
