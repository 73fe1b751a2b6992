"""The fp16 hi/lo split GEMMs (`stmp_gemm_f32`, `stmp_gemm_lstm_f32`, `stmp_gemm_blocks_f32` with EPI_BIAS) against float64 products of
the same fp32 operands, across operand magnitudes and the shape edges of the kernels, and the GConvLSTM training path at the gradient
scale of a real mean loss against the float64 oracle.

The contract checked per element.  Each fp32 operand v is split into hi = fp16(v), lo = fp16(v - hi) and the kernel accumulates
lo*hi + hi*lo + hi*hi in fp32.  With v = hi + lo + e_v, the computed product of a and w is a*w - e_a*w - a*e_w + e_a*e_w - lo_a*lo_w:
  * |lo_a*lo_w| <= 2^-22 |a||w|  (|lo| <= 2^-11 |v|);
  * |e_v| <= 2^-22 |v| + 2^-25: relative 2^-11 of lo while lo is a normal fp16 number, otherwise half of fp16's subnormal spacing 2^-24
    (this also covers hi itself rounding in the subnormal range, |v| < 2^-14, and both halves flushing to zero under 3e-8);
so a row m and column n of C = A @ W carry a split error of at most 3 * 2^-22 (|A||W|)_mn + 2^-25 (sum_k |A_mk| + sum_k |W_kn|).
The fp32 accumulation (and the bias add) adds the rounding of a float sum over K: for these zero-mean operands it stays at about
fp32's own error, which is at most 1.5 * 2^-22 (|A||W|)_mn here.  Hence the bound

    |C - C64| <= C_SPLIT * (2^-22 (|A||W| + |bias|)_mn + 2^-25 (sum_k |A_mk| + sum_k |W_kn|)),   C_SPLIT = 8  (3 + 2 * 1.5, rounded up).

The 2^-25 term is the absolute error floor of the split: callers prescale gradient-sized operands (`gconv_lstm._split_prescale`).
Inside the band where both halves are normal (|A|, |W| between about 2^-3 and 2^15) the error must also stay within 4x the CPU fp32
result's own error, the idiom of test_gpu_plan_spmm.py, where that error is a maximum over 10^5 or more elements of a K >= 32 sum.
Over a few thousand elements the maximum is too noisy a statistic, and for K = 4 fp32 rounds just three times while the split's
per-product 3 * 2^-22 dominates: the bound above still applies there."""
import ctypes

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, distributed as D, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import GConvLSTM

pytestmark = pytest.mark.gpu
DEV = "cuda"
C_SPLIT = 8.0
A_SCALES = [1e-8, 1e-6, 1e-4, 1e-2, 1.0, 1e2, 1e4]
W_SCALES = [1e-3, 1.0, 1e2]
IN_BAND = {1.0, 1e2, 1e4}


def _operands(M, K, N, sa, sw, seed, mixed=False):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g) * sa
    if mixed:                                                        # row m scaled by 10^((m mod 9) - 8): 1e-8 .. 1 in one operand
        A = A * torch.pow(10.0, (torch.arange(M) % 9 - 8).double()).float().view(M, 1)
    W = torch.randn(K, N, generator=g) * sw
    bias = torch.randn(N, generator=g)
    return A, W, bias


def _bound(A, W, bias=None):
    """Per-element error bound of the split GEMM (module docstring), float64 on the device."""
    a, w = A.double().abs(), W.double().abs()
    P = a @ w
    if bias is not None:
        P = P + bias.double().abs()
    return C_SPLIT * (2.0 ** -22 * P + 2.0 ** -25 * (a.sum(1, keepdim=True) + w.sum(0)))


def _check(got, A, W, bias, what, in_band):
    A64, W64 = A.to(DEV).double(), W.to(DEV).double()
    ref = A64 @ W64 + (0 if bias is None else bias.to(DEV).double())
    err = (got.double() - ref).abs()
    ratio = float((err / _bound(A.to(DEV), W.to(DEV), None if bias is None else bias.to(DEV))).max())
    assert bool(torch.isfinite(got).all()), what
    assert ratio <= 1.0, (what, "error / contract bound", ratio)
    if in_band and A.size(0) * W.size(1) >= 100_000 and A.size(1) >= 32:
        ref32 = (A @ W + (0 if bias is None else bias)).to(DEV).double()
        e, e32 = float(err.max()), float((ref32 - ref).abs().max())
        assert e <= 4 * e32, (what, "error vs the CPU fp32 result's own error", e, e32)


# ---- stmp_gemm_f32 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sw", W_SCALES)
@pytest.mark.parametrize("sa", A_SCALES + ["mixed"])
def test_gemm_magnitudes(sa, sw):
    M, K, N = 4097, 132, 96
    mixed = sa == "mixed"
    A, W, bias = _operands(M, K, N, 1.0 if mixed else sa, sw, seed=7, mixed=mixed)
    packed = ops.gemm_prepack(W.to(DEV))
    for b in (None, bias):
        got = ops.gemm(A.to(DEV), packed, K, N, None if b is None else b.to(DEV))
        _check(got, A, W, b, f"A~{sa} W~{sw} bias={b is not None}", sa in IN_BAND and sw in IN_BAND)


@pytest.mark.parametrize("N", [32, 96, 256])
@pytest.mark.parametrize("K", [4, 36, 68, 132, 384])
@pytest.mark.parametrize("M", [1, 127, 129, 4097])
def test_gemm_shapes(M, K, N):
    A, W, bias = _operands(M, K, N, 1.0, 1.0, seed=M * 1000 + K + N)
    packed = ops.gemm_prepack(W.to(DEV))
    c0 = _lib.path_counters().get("k_gemm_split", 0)
    got = ops.gemm(A.to(DEV), packed, K, N, bias.to(DEV))
    assert _lib.path_counters().get("k_gemm_split", 0) == c0 + 1
    _check(got, A, W, bias, (M, K, N), True)


@pytest.mark.parametrize("M,K,N,lda", [(129, 36, 96, 40), (4097, 132, 256, 196), (127, 4, 32, 8)])
def test_gemm_row_stride_and_column_view(M, K, N, lda):
    """A with a row stride lda > K (the C ABI directly: `ops.gemm` always passes lda = K) and C written through a column view of a
    wider buffer (ldc > N), as the GConvLSTM backward writes its two halves of dS.  Pad columns of A hold NaN: they must never be read;
    columns of C outside the view must keep their contents."""
    A, W, bias = _operands(M, K, N, 1.0, 1.0, seed=lda)
    Abuf = torch.full((M, lda), float("nan"), device=DEV)
    Abuf[:, :K] = A.to(DEV)
    packed = ops.gemm_prepack(W.to(DEV))
    ldc = N + 64
    Cbuf = torch.full((M, ldc), -7.0, device=DEV)
    view = Cbuf[:, 32:32 + N]
    _lib.check(_lib.lib().stmp_gemm_f32(ctypes.c_void_p(Abuf.data_ptr()), lda, M, K, N, _lib.ptr(packed), _lib.ptr(bias.to(DEV)),
                                        ctypes.c_void_p(view.data_ptr()), ldc, _lib.stream_ptr()))
    _check(view, A, W, bias, ("lda", lda), True)
    assert bool((Cbuf[:, :32] == -7).all()) and bool((Cbuf[:, 32 + N:] == -7).all())
    Cbuf.fill_(-7.0)                                                     # and through `ops.gemm(out=...)` with a dense A
    ops.gemm(A.to(DEV), packed, K, N, bias.to(DEV), out=view)
    _check(view, A, W, bias, ("out view", ldc), True)
    assert bool((Cbuf[:, :32] == -7).all()) and bool((Cbuf[:, 32 + N:] == -7).all())


# ---- stmp_gemm_blocks_f32 (EPI_BIAS) ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sw", W_SCALES)
@pytest.mark.parametrize("sa", A_SCALES + ["mixed"])
@pytest.mark.parametrize("M,widths,N", [(4097, (64, 64, 4), 96), (129, (36,), 32), (1, (64, 4), 256)])
def test_gemm_blocks_bias(M, widths, N, sa, sw):
    """The blocked GEMM (A given as K-blocks of <= 64 columns, each weight block zero-padded to 64 rows) with the plain bias epilogue."""
    K = sum(widths)
    mixed = sa == "mixed"
    A, W, bias = _operands(M, K, N, 1.0 if mixed else sa, sw, seed=11 + K, mixed=mixed)
    Ad, Wd = A.to(DEV), W.to(DEV)
    offs = [sum(widths[:i]) for i in range(len(widths))]
    blocks = [(Ad[:, o:o + w], w, 0) for o, w in zip(offs, widths)]
    packed = ops.gemm_blocks_prepack([Wd[o:o + w] for o, w in zip(offs, widths)])
    c0 = _lib.path_counters().get("k_gemm_blocks", 0)
    got = ops.gemm_blocks(blocks, packed, N, N, bias.to(DEV), ops.EPI_BIAS)
    assert _lib.path_counters().get("k_gemm_blocks", 0) == c0 + 1
    _check(got, A, W, bias, f"blocks {widths} A~{sa} W~{sw}", sa in IN_BAND and sw in IN_BAND)


# ---- stmp_gemm_lstm_f32 -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_cb", [True, False])
@pytest.mark.parametrize("cout", [32, 64])
@pytest.mark.parametrize("sa", A_SCALES + ["mixed"])
def test_gemm_lstm_magnitudes(sa, cout, with_cb):
    """The GEMM with the peephole-LSTM epilogue.  The pre-activations carry the contract bound E (per column block i, f, c, o); the gate
    chain passes it on with the sigmoid / tanh slopes (<= 1/4, <= 1) and adds the rounding of its own fp32 evaluation, 2^-20 of
    the state's scale:  E_C = |C_old| E_f / 4 + E_i / 4 + E_c,  E_H = (E_o + |w_co| E_C) / 4 + E_C."""
    M, K = 4097, 132
    mixed = sa == "mixed"
    A, W, _ = _operands(M, K, 4 * cout, 1.0 if mixed else sa, 1.0, seed=cout + K, mixed=mixed)
    g = torch.Generator().manual_seed(cout)
    cb = torch.randn(4 * cout, generator=g) if with_cb else None
    cell = torch.randn(M, cout, generator=g)
    wci, wcf, wco, bi, bf, bc, bo = (torch.randn(cout, generator=g) * 0.5 for _ in range(7))
    d = lambda t: None if t is None else t.to(DEV)
    packed = ops.gemm_prepack(W.to(DEV))
    h, c = ops.gemm_lstm(A.to(DEV), packed, K, cout, d(cb), d(cell), *map(d, (wci, wcf, wco, bi, bf, bc, bo)))
    q = lambda t: t.to(DEV).double()
    pre = q(A) @ q(W) + (0 if cb is None else q(cb))
    E = _bound(A.to(DEV), W.to(DEV), d(cb))
    pi, pf, pc, po = (pre[:, j * cout:(j + 1) * cout] for j in range(4))
    Ei, Ef, Ec, Eo = (E[:, j * cout:(j + 1) * cout] for j in range(4))
    C0 = q(cell)
    I, Fg = torch.sigmoid(pi + q(wci) * C0 + q(bi)), torch.sigmoid(pf + q(wcf) * C0 + q(bf))
    Cn = Fg * C0 + I * torch.tanh(pc + q(bc))
    Hn = torch.sigmoid(po + q(wco) * Cn + q(bo)) * torch.tanh(Cn)
    EC = C0.abs() * Ef / 4 + Ei / 4 + Ec + 2.0 ** -20 * (1 + Cn.abs())
    EH = (Eo + q(wco).abs() * EC) / 4 + EC + 2.0 ** -20
    for got, ref, bound, name in ((c, Cn, EC, "C"), (h, Hn, EH, "H")):
        ratio = float(((got.double() - ref).abs() / bound).max())
        assert ratio <= 1.0, (name, sa, cout, with_cb, ratio)


# ---- the training path at the gradient scale of a mean loss -----------------------------------------------------------------------
def test_gconv_lstm_cfg5_training_gradients_vs_float64():
    """cfg5's cell GConvLSTM(64, 64, K=3) over 12 steps on 2 000 nodes, B = 8, Linear head, masked MAE: gradients of a mean loss, 1e-6
    and below, which the fp16 split flushes unless dpre is prescaled.  Per gradient tensor the fused path's largest error against the
    float64 oracle must be at most 4x that of the op-for-op fp32 path (`fused_training = False`) plus 1e-6 of the gradient's scale."""
    n, B, T, Fd = 2000, 8, 12, 64
    ei, ew = synthetic.large_graph(n, 8000, 3)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(0)
    X = torch.randn(B, T, n, Fd, device=DEV, generator=g)
    Y = torch.randn(B, n, Fd, device=DEV, generator=g)
    Y[Y.abs() < 0.3] = 0
    torch.manual_seed(0)
    cell, head = GConvLSTM(Fd, Fd, 3).to(DEV), torch.nn.Linear(Fd, Fd).to(DEV)
    with torch.no_grad():
        for p in cell.parameters():                                      # non-zero biases and peepholes
            if p.dim() == 1 or p.size(0) == 1:
                p.normal_(0, 0.2)

    def run(fused):
        cell.fused_training = fused
        cell.zero_grad(set_to_none=True)
        head.zero_grad(set_to_none=True)
        H = C = None
        c0 = _lib.path_counters().get("k_lstm_gate_bwd", 0)
        for t in range(T):
            H, C = cell(X[:, t], ei, ew, H, C)
        D.masked_mae_loss(head(H), Y).backward()
        assert (_lib.path_counters().get("k_lstm_gate_bwd", 0) - c0 == T) == fused
        return {**{k: p.grad.clone() for k, p in cell.named_parameters()}, "head.weight": head.weight.grad.clone(),
                "head.bias": head.bias.grad.clone()}

    fused, plain = run(True), run(False)
    p = {k: v.detach().double().requires_grad_(True) for k, v in cell.state_dict().items()}
    hw, hb = (t.detach().double().requires_grad_(True) for t in (head.weight, head.bias))
    H = torch.zeros(B, n, Fd, dtype=torch.float64, device=DEV)
    C = torch.zeros_like(H)
    for t in range(T):
        H, C = R.gconv_lstm_cell(p, X[:, t].double(), ei, ew.double(), H, C)
    D.masked_mae_loss(torch.nn.functional.linear(H, hw, hb), Y.double()).backward()
    ref = {**{k: v.grad for k, v in p.items()}, "head.weight": hw.grad, "head.bias": hb.grad}
    assert float(ref["conv_x_i.lins.0.weight"].abs().max()) < 1e-3      # the mean loss: small gradients
    for k, r in ref.items():
        err = float((fused[k].double() - r).abs().max())
        base = float((plain[k].double() - r).abs().max())
        scale = float(r.abs().max())
        assert err <= 4 * base + 1e-6 * scale, (k, err, base, scale)
