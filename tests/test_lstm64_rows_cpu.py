"""Host side of GConvLSTM and GCLSTM at 64 hidden channels on the 64-wide row-split LSTM cell kernels: the routing (`_rows_ok`, whose
envelope is checked before the library or the plan's node count is consulted), the weight pack (`_rows_packed`), `ops._LstmRowsFn` and the
hand-off of the packed gradients (`_rows_spec`), with every library call replaced by a dense torch restatement of its contract
(test_lstm_rows_cpu.py's, at the width of its operands) on a dense Chebyshev plan -- predictions, costs and every gradient against the
float64 oracle, itself held to the unmodified reference (tests/golden/make_goldens_lstm64.py)."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvLSTM
from pytorch_geometric_temporal_b200.nn.recurrent import _cheb as cheb_mod
from gconvgru_seq import chickenpox_train_split
from lstm64_seq import carried_state, check_reference, load, model_for, oracle_run, run
from test_modules_host_logic_cpu import dense_graph_ops  # noqa: F401  (dense Chebyshev plan + SpMM)
from wikimaths_seq import load as load_wikimaths

MODULES = {"gconv_lstm": GConvLSTM, "gc_lstm": GCLSTM}


def _basis(plan, variant, n_ops, x, h):
    parts = [x, h]
    if n_ops:
        parts += [torch.matmul(plan.L, h)] if variant == _lib.LSTM_GC else [torch.matmul(plan.L, x), torch.matmul(plan.L, h)]
    return torch.cat(parts, -1)


def fake_pack(variant, n_ops, cin, wx, wh, bx, bh, bg):
    Co = wh.size(-1)
    blocks = []
    for g in range(4):
        if variant == _lib.LSTM_GC:
            blocks.append(torch.cat([wx[g].t()] + [wh[g, k] for k in range(n_ops + 1)], 1))
        else:
            blocks.append(torch.cat([torch.cat([wx[g, k], wh[g, k]], 1) for k in range(n_ops + 1)], 1))
    b = bg.reshape(4 * Co).clone()
    for t in (bx, bh):
        if t is not None:
            b = b + t.reshape(4 * Co)
    return torch.cat(blocks), b


def _peep(peep, Co):
    return (torch.zeros(Co) if peep is None else peep[j] for j in range(3))


def fake_fwd(plan, variant, n_ops, x, h, c, w, b, peep, train=False):
    N, Co = x.size(0), w.size(0) // 4
    h = x.new_zeros(N, Co) if h is None else h
    c = x.new_zeros(N, Co) if c is None else c
    S = _basis(plan, variant, n_ops, x, h)
    pre = S @ w.t() + b
    wci, wcf, wco = _peep(peep, Co)
    I, F = torch.sigmoid(pre[:, :Co] + wci * c), torch.sigmoid(pre[:, Co:2 * Co] + wcf * c)
    T = torch.tanh(pre[:, 2 * Co:3 * Co])
    cn = F * c + I * T
    O = torch.sigmoid(pre[:, 3 * Co:] + wco * cn)
    hn = O * torch.tanh(cn)
    return (hn, cn, torch.stack([I, F, T, O]), S) if train else (hn, cn)


def fake_bwd(plan, variant, n_ops, gh, gc, c, cn, stash, w, peep, want_dx, want_dh, want_dc, cin):
    I, F, T, O = stash
    Co = cn.size(1)
    cp = torch.zeros_like(cn) if c is None else c
    g = torch.zeros_like(cn) if gh is None else gh
    gcv = torch.zeros_like(cn) if gc is None else gc
    wci, wcf, wco = _peep(peep, Co)
    tc = torch.tanh(cn)
    dpo = g * tc * O * (1 - O)
    dcn = gcv + g * O * (1 - tc * tc) + dpo * wco
    dpi, dpf, dpc = dcn * T * I * (1 - I), dcn * cp * F * (1 - F), dcn * I * (1 - T * T)
    dpre = torch.cat([dpi, dpf, dpc, dpo], 1)
    dS = dpre @ w
    C = cin + Co
    dx, dh = dS[:, :cin].clone(), dS[:, cin:C].clone()
    if n_ops:
        LT = plan.L.t()
        if variant == _lib.LSTM_GC:
            dh += LT @ dS[:, C:]
        else:
            dx += LT @ dS[:, C:C + cin]
            dh += LT @ dS[:, C + cin:]
    dc = dcn * F + dpi * wci + dpf * wcf
    return (torch.stack([dpre[:, :2 * Co], dpre[:, 2 * Co:]]), dx if want_dx else None, dh if want_dh else None,
            dc if want_dc else None, (cp, cn))


def fake_wgrad(variant, n_ops, cin, S, dpre, scratch, has_peep):
    d = torch.cat([dpre[0], dpre[1]], 1)
    Co = d.size(1) // 4
    cp, cn = scratch
    peep = torch.cat([(d[:, :Co] * cp).sum(0), (d[:, Co:2 * Co] * cp).sum(0), (d[:, 3 * Co:] * cn).sum(0)])
    return d.t() @ S, torch.cat([d.sum(0), peep if has_peep else torch.full((3 * Co,), float("nan"))])


class _Plan(object):
    def __init__(self, L):
        self.L, self.num_nodes = L, L.size(0)


@pytest.fixture()
def dense_rows(dense_graph_ops, monkeypatch):   # noqa: F811
    calls = []
    dense = cheb_mod.ChebPlanMixin._cheb_plan
    monkeypatch.setattr(cheb_mod.ChebPlanMixin, "_cheb_plan", lambda self, *a, **k: _Plan(dense(self, *a, **k).L))

    def counted(name, fn):
        def f(*a, **k):
            calls.append(name)
            return fn(*a, **k)
        return f
    monkeypatch.setattr(ops, "_require_cuda", lambda *a, **k: None)
    monkeypatch.setattr(ops, "lstm_rows_supported", counted("supported", lambda plan, variant, n_ops, cin, cout: n_ops <= 1 and cin <= 16
                                                             and cout in (32, 64)))
    monkeypatch.setattr(ops, "lstm_rows_pack_weights", counted("pack", fake_pack))
    monkeypatch.setattr(ops, "lstm_rows_fwd", counted("fwd", fake_fwd))
    monkeypatch.setattr(ops, "lstm_rows_bwd", counted("bwd", fake_bwd))
    monkeypatch.setattr(ops, "lstm_rows_wgrad", counted("wgrad", fake_wgrad))
    return calls


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().double(), want.detach().double()
    assert got.shape == want.shape and torch.allclose(got, want, rtol=rtol, atol=atol), float((got - want).abs().max())


@pytest.mark.parametrize("case", ["K2_sym", "K1_sym", "K2_rw", "K2_sym_carried", "chickenpox"])
@pytest.mark.parametrize("name", list(MODULES))
def test_host_logic_vs_reference_golden(golden_dir, dense_rows, name, case):
    c = load(golden_dir)["cases"][f"{name}/{case}"]
    if case == "chickenpox":
        ei, ew, X, Y = chickenpox_train_split()
    else:
        g = load_wikimaths(golden_dir)
        ei, ew, X, Y = g["edge_index"], g["edge_weight"], g["X"], g["Y"]
    m = model_for(c, fused=True)
    n = X.size(1)
    carried = "gH0" in c["fingerprints"]
    H0 = carried_state(n, 7, 13, 17).requires_grad_(True) if carried else None
    C0 = carried_state(n, 5, 11, 19).requires_grad_(True) if carried else None
    H064 = None if H0 is None else H0.detach().double().requires_grad_(True)
    C064 = None if C0 is None else C0.detach().double().requires_grad_(True)
    out64, cost64, leaves = oracle_run(c, X, Y, ei, ew, c["lambda_max"], H064, C064)
    cost64.backward()
    check_reference(c, out64, cost64, {k: v.grad for k, v in leaves.items()}, *((H064.grad, C064.grad) if carried else ()))
    out, cost = run(m, X, Y, ei, ew, c["lambda_max"], H0, C0)
    cost.backward()
    _close(out, out64)
    _close(cost, cost64, 1e-5, 1e-7)
    for k, p in m.named_parameters():
        _close(p.grad, leaves[k].grad, 1e-3, 1e-3 * float(leaves[k].grad.abs().max()) + 1e-6)
    if carried:
        _close(H0.grad, H064.grad, 1e-3, 1e-3 * float(H064.grad.abs().max()))
        _close(C0.grad, C064.grad, 1e-3, 1e-3 * float(C064.grad.abs().max()))
    S = X.size(0)
    assert [k for k in dense_rows if k != "supported"] == ["pack"] + ["fwd"] * S + ["bwd", "wgrad"] * S


def test_pack_and_spec_layouts_at_64(dense_rows):
    """The packed weights are the gate weights in basis order at 64 rows per gate, and every spec block is where the pack put the
    parameter: a packed gradient made of the pack itself hands each parameter back its own value."""
    torch.manual_seed(0)
    for K, cin, bias in ((2, 14, True), (1, 16, True), (2, 3, False)):
        m = GConvLSTM(cin, 64, K, bias=bias)
        w, b, peep = m._rows_packed()
        assert w.shape == (256, K * (cin + 64)) and torch.equal(w, m._weight().t())
        want = torch.cat([getattr(m, f"b_{g}").reshape(64) for g in "ifco"])
        if bias:
            want = m._conv_bias() + want
        assert torch.allclose(b, want) and peep.shape == (3, 64) and torch.equal(peep, torch.cat([m.w_c_i, m.w_c_f, m.w_c_o]))
        spec, params = m._rows_spec()
        assert len(spec) == len(params) == len(list(m.parameters()))
        dbp = torch.cat([torch.zeros(256), peep.reshape(-1)])
        for (kind, *s), p, got in zip(spec, params, ops._spec_grads(spec, w, dbp)):
            if kind == "w":
                assert torch.equal(got, p), s
            elif s[0] >= 256:                                          # the peepholes sit behind the 256 summed biases
                assert torch.equal(got.reshape(p.shape), p), s
        g = GCLSTM(cin, 64, K, bias=bias)
        w, b = g._rows_packed()
        assert w.shape == (256, cin + 64 * K) and torch.equal(w, g._weight().t())
        assert torch.allclose(b, torch.cat(g._gate_bias()))
        spec, params = g._rows_spec()
        for (kind, *s), p, got in zip(spec, params, ops._spec_grads(spec, w, torch.zeros(256))):
            if kind in ("w", "wt"):
                assert torch.equal(got, p), s


def test_routing(dense_rows, monkeypatch):
    """The module's envelope is checked before the library is asked; inference with in_channels % 4 == 0 leaves the 64-wide cell from
    ops.LSTM_WIDE_ROWS_GEMM_NODES nodes on (the node count comes from the plan), training never does; the 32-wide routes are unchanged."""
    ei, ew, X, _ = chickenpox_train_split()
    x = X[0]
    for cls in MODULES.values():
        dense_rows.clear()
        for m, xx in ((cls(17, 64, 2), torch.randn(20, 17)), (cls(4, 64, 3), x), (cls(4, 64, 2), x.expand(2, 20, 4))):
            assert not m._rows_ok(m._cheb_plan(ei, ew, 20, "sym", None), xx, None, None, True)
            assert not m._rows_ok(m._cheb_plan(ei, ew, 20, "sym", None), xx, None, None, False)
        m = cls(4, 64, 2)
        plan = m._cheb_plan(ei, ew, 20, "sym", None)
        assert not m._rows_ok(plan, x, torch.zeros(20, 32), None, True)          # a state of the wrong width
        assert not m._rows_ok(plan, x.double(), None, None, True)
        assert dense_rows == [], dense_rows                           # none of these consulted the library
        m.fused_training = False
        assert not m._rows_ok(plan, x, None, None, True) and m._rows_ok(plan, x, None, None, False)
        m.fused_training = True
        assert m._rows_ok(plan, x, None, None, True)
        big = ops.LSTM_WIDE_ROWS_GEMM_NODES
        for n, cin, training, want in ((big - 1, 4, False, True), (big, 4, False, False), (big, 16, False, False), (big, 5, False, True),
                                       (big, 4, True, True)):
            m = cls(cin, 64, 2)
            p = _Plan(torch.zeros(1, 1))
            p.num_nodes = n
            assert m._rows_ok(p, torch.zeros(n, cin), None, None, training) == want, (cls, n, cin, training)
        m = cls(4, 32, 2)                                             # 32 wide: no node-count rule
        p.num_nodes = 10 * big
        assert m._rows_ok(p, torch.zeros(p.num_nodes, 4), None, None, False)
