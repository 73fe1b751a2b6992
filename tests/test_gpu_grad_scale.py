"""Loss-scale equivariance of every fused training backward: the backward is linear in dL/dout, so a loss multiplied by an exact power
of two, 2^-24 or 2^+8, must give every gradient multiplied by the same power of two, bit for bit.

fp32 FFMA arithmetic commutes exactly with a power-of-two scale as long as nothing leaves the normal range, and so does the TF32 hi/lo
split of the weight-gradient contraction (TF32 keeps fp32's exponent).  An fp16 hi/lo split does not: its halves go subnormal below
2^-14 and vanish below 3e-8, which is where the gradients of a mean loss live.  A path that feeds gradients to such a split must bring
them into range with an exact power of two derived from their own maximum (as `gconv_lstm._split_prescale` does), and then it is
equivariant too.  Each case uses a realistic mean loss (masked MAE through `distributed.masked_mae_loss`), so the unscaled gradients are
already small, and checks with the path counters that the fused kernels served every call."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, distributed as D
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN2, TGCN2, BatchedDCRNN, GConvLSTM

pytestmark = pytest.mark.gpu
DEV = "cuda"
EXPONENTS = (-24, 8)


def _graph(seed=0):
    ei, ew, _ = synthetic.metr_la_like(seed, 16)
    return torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)


def _targets(*shape, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    Y = torch.randn(*shape, device=DEV, generator=g)
    Y[Y.abs() < 0.2] = 0                                             # missing readings, as in the traffic datasets
    return Y


def _with_bias(m, seed):
    torch.manual_seed(seed)
    with torch.no_grad():
        for p in m.parameters():                                     # non-zero biases: a bias-gradient mistake cannot hide
            if p.dim() == 1 or p.size(0) == 1:
                p.normal_(0, 0.2)
    return m.to(DEV)


def _ran(c0):
    c1 = _lib.path_counters()
    return {k: v - c0.get(k, 0) for k, v in c1.items() if v > c0.get(k, 0)}


def _grads(params, X=None):
    out = {k: p.grad.clone() for k, p in params}
    if X is not None:
        out["X"] = X.grad.clone()
    return out


def _assert_equivariant(run):
    """run(scale) -> {name: gradient} of `scale * loss`; every gradient of 2^e * loss is 2^e times that of the loss, bit for bit."""
    base = run(1.0)
    for k, g in base.items():
        assert bool(torch.isfinite(g).all()), k
    # a gradient may be exactly zero (the r gate of a TGCN step without an incoming state has nothing to act on), but not all of them
    assert sum(float(g.abs().max()) > 0 for g in base.values()) > len(base) // 2
    for e in EXPONENTS:
        got = run(2.0 ** e)
        for k, g in base.items():
            want = g * 2.0 ** e
            if not torch.equal(got[k], want):
                bad = got[k] != want
                rel = float(((got[k] - want).abs().max()) / want.abs().max())
                pytest.fail(f"2^{e} * loss: gradient {k} differs from 2^{e} x gradient in {int(bad.sum())} of {bad.numel()} elements, "
                            f"largest by {rel:.3e} of its scale")


class _Options:
    """Sets library switches for a block and restores their defaults (all 1) afterwards."""

    def __init__(self, **opts):
        self.opts = opts

    def __enter__(self):
        for k, v in self.opts.items():
            _lib.set_option(k, v)

    def __exit__(self, *exc):
        for k in self.opts:
            _lib.set_option(k, 1)


@pytest.mark.parametrize("bwd_split", [1, 0])
@pytest.mark.parametrize("wgrad_tc", [1, 0])
def test_dcrnn_fused_backward(wgrad_tc, bwd_split):
    """BatchedDCRNN(2, 32, 2): the persistent reverse-time kernel k_dcrnn_bwd_seq (on a 2-CTA cluster per window or one CTA) and the
    weight gradients on wgmma with the TF32 split (k_dcrnn_wgrad_tc) or on FFMA (k_dcrnn_wgrad)."""
    ei, ew = _graph()
    m = _with_bias(BatchedDCRNN(2, 32, 2), 0)
    X0 = torch.randn(4, 12, 207, 2, device=DEV)
    Y = _targets(4, 12, 207, 32)
    wgrad = "k_dcrnn_wgrad_tc" if wgrad_tc else "k_dcrnn_wgrad"

    def run(scale):
        m.zero_grad(set_to_none=True)
        X = X0.clone().requires_grad_(True)
        with _Options(dcrnn_wgrad_tc=wgrad_tc, dcrnn_bwd_split=bwd_split):
            c0 = _lib.path_counters()
            (D.masked_mae_loss(m(X, ei, ew), Y) * scale).backward()
            ran = _ran(c0)
        assert ran.get("k_dcrnn_seq_tc") == 1 and ran.get("k_dcrnn_bwd_seq") == 1 and ran.get("k_masked_mae_bwd") == 1
        assert ran.get("k_dcrnn_bwd_seq[cluster2]", 0) == bwd_split
        assert ran.get(wgrad, 0) >= 1 and ran.get("k_dcrnn_wgrad_tc" if not wgrad_tc else "k_dcrnn_wgrad", 0) == 0
        return _grads(m.named_parameters(), X)
    _assert_equivariant(run)


def test_dcrnn_narrow_fused_backward():
    """BatchedDCRNN(2, 2, 3), the reference's index-batching training model: k_dcrnn_narrow_bwd."""
    ei, ew = _graph(1)
    m = _with_bias(BatchedDCRNN(2, 2, 3), 1)
    X0 = torch.randn(4, 12, 207, 2, device=DEV)
    Y = _targets(4, 12, 207, 2)

    def run(scale):
        m.zero_grad(set_to_none=True)
        X = X0.clone().requires_grad_(True)
        c0 = _lib.path_counters()
        (D.masked_mae_loss(m(X, ei, ew), Y) * scale).backward()
        ran = _ran(c0)
        assert ran.get("k_dcrnn_narrow_seq") == 1 and ran.get("k_dcrnn_narrow_bwd") == 1
        return _grads(m.named_parameters(), X)
    _assert_equivariant(run)


def test_a3tgcn2_fused_backward():
    """A3TGCN2(2, 32, 12) and A3TGCN2(1, 32, 128) (four 32-period chunks per lane) without an incoming state under a Linear head:
    k_tgcn_attn_bwd."""
    ei, ew = _graph(2)
    head = torch.nn.Linear(32, 12).to(DEV)
    Y = _targets(8, 207, 12)
    for fin, periods in ((2, 12), (1, 128)):
        m = _with_bias(A3TGCN2(fin, 32, periods, 8), 2)
        X = torch.randn(8, 207, fin, periods, device=DEV)

        def run(scale):
            m.zero_grad(set_to_none=True)
            head.zero_grad(set_to_none=True)
            c0 = _lib.path_counters()
            (D.masked_mae_loss(head(torch.relu(m(X, ei, ew))), Y) * scale).backward()
            ran = _ran(c0)
            assert ran.get("k_tgcn_attn_bwd") == 1
            return _grads(list(m.named_parameters()) + [("head." + k, p) for k, p in head.named_parameters()])
        _assert_equivariant(run)


def test_tgcn2_carried_state_fused_backward():
    """The reference's BatchedTGCN loop: TGCN2(2, 32, 1) once per step over 12 steps with the state carried, ReLU, Linear head.
    Step 0 runs k_tgcn_attn_bwd, steps 1..11 k_tgcn_cell_bwd."""
    ei, ew = _graph(3)
    m = _with_bias(TGCN2(2, 32, 1), 3)
    head = torch.nn.Linear(32, 2).to(DEV)
    X = torch.randn(8, 207, 2, 12, device=DEV)
    Y = _targets(8, 12, 207, 2)

    def run(scale):
        m.zero_grad(set_to_none=True)
        head.zero_grad(set_to_none=True)
        c0 = _lib.path_counters()
        h, outs = None, []
        for t in range(12):
            h = m(X[..., t], ei, ew, h)
            outs.append(head(torch.relu(h)))
        (D.masked_mae_loss(torch.stack(outs, 1), Y) * scale).backward()
        ran = _ran(c0)
        assert ran.get("k_tgcn_attn_bwd") == 1 and ran.get("k_tgcn_cell_bwd") == 11 and "k_spmm" not in ran
        return _grads(list(m.named_parameters()) + [("head." + k, p) for k, p in head.named_parameters()])
    _assert_equivariant(run)


def test_gconv_lstm_fused_backward():
    """cfg5's cell GConvLSTM(64, 64, K=3) over 12 steps under a Linear head: the hand-written `_LstmCellFn` backward, whose
    dS = dpre @ W^T runs on the fp16-split wgmma GEMM.  Without the power-of-two prescale of dpre the split flushes these gradients."""
    ei, ew = synthetic.large_graph(1000, 5000, 4)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    cell = _with_bias(GConvLSTM(64, 64, 3), 4)
    head = torch.nn.Linear(64, 64).to(DEV)
    X0 = torch.randn(4, 12, 1000, 64, device=DEV)
    Y = _targets(4, 1000, 64)

    def run(scale):
        cell.zero_grad(set_to_none=True)
        head.zero_grad(set_to_none=True)
        X = X0.clone().requires_grad_(True)
        c0 = _lib.path_counters()
        H = C = None
        for t in range(12):
            H, C = cell(X[:, t], ei, ew, H, C)
        (D.masked_mae_loss(head(H), Y) * scale).backward()
        ran = _ran(c0)
        assert ran.get("k_lstm_gate_bwd") == 12 and ran.get("k_gemm_split", 0) >= 12 * 4
        return _grads(list(cell.named_parameters()) + [("head." + k, p) for k, p in head.named_parameters()], X)
    _assert_equivariant(run)


def test_masked_mae_backward():
    """stmp_masked_mae_bwd on its own, with missing targets."""
    pred0 = torch.randn(8, 12, 325, 2, device=DEV)
    Y = _targets(8, 12, 325, 2)

    def run(scale):
        pred = pred0.clone().requires_grad_(True)
        c0 = _lib.path_counters()
        (D.masked_mae_loss(pred, Y) * scale).backward()
        assert _ran(c0).get("k_masked_mae_bwd") == 1
        return {"pred": pred.grad}
    _assert_equivariant(run)
