"""Host side of the 64-wide fused TGCN / A3TGCN path (the stmp_tgcn_wide_* entries): the folded-weight layouts `TGCN._packed3` and
`TGCN._fold3` at 64 hidden channels, the routing of every call between the fused kernels and the op-for-op path, and the weight-gradient
layout of the 64-wide cell backward (the contraction's dw [192][fin + 64] over the bases [A^X | H], [A^X | H*R], transposed into dA, dBm
and dc), with the kernels replaced by dense differentiable restatements of their arithmetic."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN, A3TGCN2, TGCN, TGCN2
from test_modules_host_logic_cpu import dense_dconv_gcn_ops  # noqa: F401  (dense GCN plan + SpMM, no fused inference kernels)
from tgcn64_seq import CASES, check_reference, data, load, model_for, oracle_run, run


def _model(cls, *args, seed=0):
    torch.manual_seed(seed)
    m = cls(*args)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.normal_(0, 0.5)
    return m


def _graph(n=23, seed=0):
    g = torch.Generator().manual_seed(seed)
    src = torch.cat([torch.arange(n), torch.randint(0, n, (3 * n,), generator=g)])
    dst = torch.cat([(torch.arange(n) + 1) % n, torch.randint(0, n, (3 * n,), generator=g)])
    keep = src != dst
    return torch.stack([src[keep], dst[keep]]), torch.rand(int(keep.sum()), generator=g) + 0.1


def _pre(m, ax, hz, hh):
    """The module's own gate pre-activations [z | r | h] from A^X: L_g [A^X W_g^T + b_g | H'] + l_g, H' = hz for z and r, hh for h."""
    out = []
    for g, hp in zip("zrh", (hz, hz, hh)):
        conv, lin = getattr(m, f"conv_{g}"), getattr(m, f"linear_{g}")
        out.append(torch.nn.functional.linear(torch.cat([ax @ conv.lin.weight.t() + conv.bias, hp], -1), lin.weight, lin.bias))
    return out


def _folded_pre(A, Bm, c, ax, hz, hh, w):
    return [ax @ A[:, w * g:w * g + w] + hp @ Bm[:, w * g:w * g + w] + c[w * g:w * g + w] for g, hp in enumerate((hz, hz, hh))]


@pytest.mark.parametrize("fin", [1, 2, 3, 4])
def test_packed3_and_fold3_at_64(fin):
    m = _model(TGCN, fin, 64, seed=fin)
    A, Bm, c = m._packed3()
    assert A.shape == (fin, 192) and Bm.shape == (64, 192) and c.shape == (192,)
    Af, Bf, cf = m._fold3()
    assert torch.equal(A, Af.detach()) and torch.equal(Bm, Bf.detach()) and torch.equal(c, cf.detach())
    g = torch.Generator().manual_seed(fin)
    ax, hz, hh = torch.randn(9, fin, generator=g), torch.randn(9, 64, generator=g), torch.randn(9, 64, generator=g)
    with torch.no_grad():
        for got, want in zip(_folded_pre(A, Bm, c, ax, hz, hh, 64), _pre(m, ax, hz, hh)):
            assert torch.allclose(got, want, rtol=1e-5, atol=1e-5)


def test_32_wide_layout_is_unchanged():
    """At out_channels 32 the blocks stay 32 columns wide, and a narrower module keeps its 32-column slots zero-padded."""
    m = _model(TGCN, 2, 32)
    A, Bm, c = m._packed3()
    assert A.shape == (2, 96) and Bm.shape == (32, 96) and c.shape == (96,)
    Af, Bf, cf = m._fold3()
    assert torch.equal(A, Af.detach()) and torch.equal(Bm, Bf.detach()) and torch.equal(c, cf.detach())
    A, Bm, c = _model(TGCN, 2, 16)._packed3()
    assert A.shape == (2, 96) and Bm.shape == (32, 96)
    for g in range(3):
        assert not A[:, 32 * g + 16:32 * g + 32].any() and not Bm[16:].any() and not c[32 * g + 16:32 * g + 32].any()


def _gates(L, x, h, A, Bm, c, probs=None):
    """The fused kernels' arithmetic, densely: out = sum_t probs[t] GRU((A^X)_t, h) at the width Bm.shape[0]."""
    w = Bm.shape[0]
    out = 0
    for t in range(x.shape[-1]):
        ax = torch.matmul(L, x[..., t])
        pz, pr, _ = _folded_pre(A, Bm, c, ax, h, h, w)
        Z, R = torch.sigmoid(pz), torch.sigmoid(pr)
        ph = _folded_pre(A, Bm, c, ax, h, h * R, w)[2]
        hn = Z * h + (1 - Z) * torch.tanh(ph)
        out = out + (hn if probs is None else probs[t] * hn)
    return out


@pytest.fixture()
def dense_kernels(dense_dconv_gcn_ops, monkeypatch):   # noqa: F811
    calls = []

    def fake_fwd(plan, x, A, Bm, c, probs=None, h=None, h_shared=False):
        calls.append(("fwd", Bm.shape[0], tuple(x.shape)))
        hh = torch.zeros(*x.shape[:2], Bm.shape[0]) if h is None else (h.expand(x.shape[0], *h.shape) if h_shared else h)
        return _gates(plan.mats[0], x, hh, A, Bm, c, probs)

    def fake_attn_train(plan, x, A, Bm, c, probs=None):
        calls.append(("attn", Bm.shape[0], tuple(x.shape)))
        return _gates(plan.mats[0], x, torch.zeros(*x.shape[:2], Bm.shape[0]), A, Bm, c, probs)

    def fake_cell_train(plan, x, h, A, Bm, c):
        calls.append(("cell", Bm.shape[0], tuple(x.shape), tuple(h.shape)))
        return _gates(plan.mats[0], x, h, A, Bm, c)
    monkeypatch.setattr(ops, "tgcn_attn_fwd", fake_fwd)
    monkeypatch.setattr(ops, "tgcn_attn_train", fake_attn_train)
    monkeypatch.setattr(ops, "tgcn_cell_train", fake_cell_train)
    return calls


def test_routing_at_64(dense_kernels):
    ei, ew = _graph()
    n, B = 23, 2
    g = torch.Generator().manual_seed(1)
    X, H = torch.randn(B, n, 2, generator=g), 0.5 * torch.randn(B, n, 64, generator=g)
    m = _model(TGCN2, 2, 64, B)
    with torch.no_grad():
        m(X, ei, ew, H)
        m(X, ei, ew)
    m(X, ei, ew).sum().backward()                                              # first step: the H = None pair
    m(X, ei, ew, H).sum().backward()                                           # carried state: the cell backward
    _model(TGCN, 2, 64)(X[0], ei, ew, H[0]).sum().backward()
    a2 = _model(A3TGCN2, 2, 64, 12, B)
    a2(torch.randn(B, n, 2, 12), ei, ew).sum().backward()
    a1 = _model(A3TGCN, 4, 64, 4)
    with torch.no_grad():
        a1(torch.randn(n, 4, 4), ei, ew, H[0])                                 # one state shared by every period
    assert dense_kernels == [("fwd", 64, (B, n, 2, 1)), ("fwd", 64, (B, n, 2, 1)), ("attn", 64, (B, n, 2, 1)),
                             ("cell", 64, (B, n, 2, 1), (B, n, 64)), ("cell", 64, (1, n, 2, 1), (1, n, 64)),
                             ("attn", 64, (B, n, 2, 12)), ("fwd", 64, (1, n, 4, 4))]


def test_calls_outside_the_64_wide_envelope_stay_op_for_op(dense_kernels):
    ei, ew = _graph()
    n, B = 23, 2
    g = torch.Generator().manual_seed(2)
    X, H = torch.randn(B, n, 2, generator=g), 0.5 * torch.randn(B, n, 64, generator=g)
    Xg = X.clone().requires_grad_(True)
    _model(TGCN2, 2, 64, B)(Xg, ei, ew, H).sum().backward()                    # gradient w.r.t. X
    assert Xg.grad is not None
    _model(TGCN2, 2, 48, B)(X, ei, ew, H[..., :48]).sum().backward()           # out_channels 48
    with torch.no_grad():
        _model(TGCN2, 2, 48, B)(X, ei, ew, H[..., :48])
    _model(TGCN2, 5, 64, B)(torch.randn(B, n, 5), ei, ew, H).sum().backward()  # in_channels 5
    _model(A3TGCN2, 2, 64, 65, B)(torch.randn(B, n, 2, 65), ei, ew).sum().backward()     # in_channels * periods 130
    Hg = H.clone().requires_grad_(True)
    _model(A3TGCN2, 2, 64, 4, B)(torch.randn(B, n, 2, 4), ei, ew, Hg).sum().backward()   # A3TGCN training with a state
    assert Hg.grad is not None
    m = _model(TGCN2, 2, 64, B)
    m.fused_training = False
    m(X, ei, ew, H).sum().backward()
    assert dense_kernels == []
    with torch.no_grad():                                                      # batch rows past one launch's grid
        assert not TGCN2(2, 64, 1)._attn_ok(X, None, 1, TGCN._FUSED_MAX_ROWS + 1)
        assert TGCN2(2, 64, 1)._attn_ok(X, None, 1, TGCN._FUSED_MAX_ROWS)


@pytest.mark.parametrize("fin", [1, 4])
def test_weight_gradient_layout_of_the_cell_backward(fin):
    """The 64-wide cell backward contracts the per-row gate gradients dp = [dpz | dpr | dph] with S1 = [A^X | H] (z, r) and
    S2 = [A^X | H*R] (h) into dw [192][fin + 64] (row = gate column, column = basis column) and db = 1^T dp; k_tgcn_wide_wgrad_unpack
    takes dA = dw[:, :fin]^T and dBm = dw[:, fin:]^T.  That is autograd's gradient of sum(pre * dp) w.r.t. A, Bm and c."""
    rows = 37
    g = torch.Generator().manual_seed(fin)
    ax, h, R, dp = (torch.randn(rows, fin, generator=g), torch.randn(rows, 64, generator=g), torch.rand(rows, 64, generator=g),
                    torch.randn(rows, 192, generator=g))
    A, Bm, c = (torch.randn(*s, generator=g).requires_grad_(True) for s in ((fin, 192), (64, 192), (192,)))
    pre = torch.cat(_folded_pre(A, Bm, c, ax, h, h * R, 64), -1)
    (pre * dp).sum().backward()
    S1, S2 = torch.cat([ax, h], -1), torch.cat([ax, h * R], -1)
    dw = torch.cat([dp[:, :64].t() @ S1, dp[:, 64:128].t() @ S1, dp[:, 128:].t() @ S2])       # k_wide_rows_wgrad<3> + its reduce
    assert dw.shape == (192, fin + 64)
    assert torch.allclose(dw[:, :fin].t(), A.grad, rtol=1e-5, atol=1e-4)
    assert torch.allclose(dw[:, fin:].t(), Bm.grad, rtol=1e-5, atol=1e-4)
    assert torch.allclose(dp.sum(0), c.grad, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("name", list(CASES))
def test_goldens_host_logic_vs_reference(golden_dir, dense_kernels, name):
    """The float64 oracle reproduces the unmodified reference's fingerprints, and the module's host logic over the dense restatement of
    the 64-wide kernels matches the oracle: outputs, loss and every gradient."""
    c = load(golden_dir)[name]
    d = data(c)
    out, loss, grads, extra = oracle_run(c, d)
    check_reference(c, out, loss, grads, extra)
    got = run(model_for(c), c, d)
    assert torch.allclose(got["out"].double(), out, rtol=1e-4, atol=1e-5)
    if loss is not None:
        assert abs(float(got["loss"].detach()) - float(loss.detach())) <= 1e-4 * abs(float(loss.detach())) + 1e-6
        for k, g in {**grads, **extra}.items():
            want = g.double()
            mine = (got["grads"][k] if k in grads else got[k]).double()
            assert torch.allclose(mine, want, rtol=1e-3, atol=1e-3 * float(want.abs().max()) + 1e-6), k
    assert {t[0] for t in dense_kernels} <= {"fwd", "attn", "cell"} and dense_kernels
