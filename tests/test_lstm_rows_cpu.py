"""Host side of GConvLSTM and GCLSTM on the row-split LSTM cell kernel (stmp_lstm_rows_*): the routing of a call (`_rows_ok`), the weight
pack (`_rows_packed`), the autograd Function `ops._LstmRowsFn` with either output's gradient absent, and the hand-off of the packed
gradients to the parameters (`_rows_spec`, `ops._spec_grads`), with every library call replaced by a dense torch restatement of its
contract on a dense Chebyshev plan -- outputs, costs and EVERY gradient against the unmodified reference on the chickenpox tutorial
(tests/golden/make_goldens_lstm.py)."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvLSTM
from test_modules_host_logic_cpu import dense_graph_ops  # noqa: F401  (dense Chebyshev plan + SpMM)
import lstm_seq

CASES = [f"{m}_chickenpox_{k}" for m in ("gconvlstm", "gclstm") for k in ("K1_sym", "K2_sym", "K2_rw")]


def _basis(plan, variant, n_ops, x, h):
    parts = [x, h]
    if n_ops:
        parts += [torch.matmul(plan.L, h)] if variant == _lib.LSTM_GC else [torch.matmul(plan.L, x), torch.matmul(plan.L, h)]
    return torch.cat(parts, -1)


def fake_pack(variant, n_ops, cin, wx, wh, bx, bh, bg):
    blocks = []
    for g in range(4):
        if variant == _lib.LSTM_GC:
            blocks.append(torch.cat([wx[g].t()] + [wh[g, k] for k in range(n_ops + 1)], 1))
        else:
            blocks.append(torch.cat([torch.cat([wx[g, k], wh[g, k]], 1) for k in range(n_ops + 1)], 1))
    b = bg.reshape(128).clone()
    for t in (bx, bh):
        if t is not None:
            b = b + t.reshape(128)
    return torch.cat(blocks), b


def _gates(pre, c, peep):
    wci, wcf, wco = (torch.zeros(32) if peep is None else peep[j] for j in range(3))
    I, F = torch.sigmoid(pre[:, :32] + wci * c), torch.sigmoid(pre[:, 32:64] + wcf * c)
    T = torch.tanh(pre[:, 64:96])
    cn = F * c + I * T
    O = torch.sigmoid(pre[:, 96:] + wco * cn)
    return I, F, T, O, cn


def fake_fwd(plan, variant, n_ops, x, h, c, w, b, peep, train=False):
    N = x.size(0)
    h = x.new_zeros(N, 32) if h is None else h
    c = x.new_zeros(N, 32) if c is None else c
    S = _basis(plan, variant, n_ops, x, h)
    I, F, T, O, cn = _gates(S @ w.t() + b, c, peep)
    hn = O * torch.tanh(cn)
    return (hn, cn, torch.stack([I, F, T, O]), S) if train else (hn, cn)


def fake_bwd(plan, variant, n_ops, gh, gc, c, cn, stash, w, peep, want_dx, want_dh, want_dc, cin):
    I, F, T, O = stash
    cp = torch.zeros_like(cn) if c is None else c
    g = torch.zeros_like(cn) if gh is None else gh
    gcv = torch.zeros_like(cn) if gc is None else gc
    wci, wcf, wco = (torch.zeros(32) if peep is None else peep[j] for j in range(3))
    tc = torch.tanh(cn)
    dpo = g * tc * O * (1 - O)
    dcn = gcv + g * O * (1 - tc * tc) + dpo * wco
    dpi, dpf, dpc = dcn * T * I * (1 - I), dcn * cp * F * (1 - F), dcn * I * (1 - T * T)
    dpre = torch.cat([dpi, dpf, dpc, dpo], 1)
    dS = dpre @ w
    C = cin + 32
    dx, dh = dS[:, :cin].clone(), dS[:, cin:C].clone()
    if n_ops:
        LT = plan.L.t()
        if variant == _lib.LSTM_GC:
            dh += LT @ dS[:, C:]
        else:
            dx += LT @ dS[:, C:C + cin]
            dh += LT @ dS[:, C + cin:]
    dc = dcn * F + dpi * wci + dpf * wcf
    return (torch.stack([dpre[:, :64], dpre[:, 64:]]), dx if want_dx else None, dh if want_dh else None, dc if want_dc else None,
            (cp, cn))


def fake_wgrad(variant, n_ops, cin, S, dpre, scratch, has_peep):
    d = torch.cat([dpre[0], dpre[1]], 1)
    cp, cn = scratch
    peep = torch.cat([(d[:, :32] * cp).sum(0), (d[:, 32:64] * cp).sum(0), (d[:, 96:] * cn).sum(0)])
    return d.t() @ S, torch.cat([d.sum(0), peep if has_peep else torch.full((96,), float("nan"))])


@pytest.fixture()
def dense_rows(dense_graph_ops, monkeypatch):   # noqa: F811
    calls = []

    def counted(name, fn):
        def f(*a, **k):
            calls.append(name)
            return fn(*a, **k)
        return f
    monkeypatch.setattr(ops, "_require_cuda", lambda *a, **k: None)
    monkeypatch.setattr(ops, "lstm_rows_supported", lambda plan, variant, n_ops, cin, cout: n_ops <= 1 and cin <= 16 and cout == 32)
    monkeypatch.setattr(ops, "lstm_rows_pack_weights", counted("pack", fake_pack))
    monkeypatch.setattr(ops, "lstm_rows_fwd", counted("fwd", fake_fwd))
    monkeypatch.setattr(ops, "lstm_rows_bwd", counted("bwd", fake_bwd))
    monkeypatch.setattr(ops, "lstm_rows_wgrad", counted("wgrad", fake_wgrad))
    return calls


def _check_grads(m, c):
    for k, p in m.named_parameters():
        ref = c["grads"][k]
        assert p.grad is not None, k
        assert p.grad.shape == ref.shape, k
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-6), k


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", CASES)
def test_chickenpox_host_logic_vs_reference_golden(golden_dir, dense_rows, case, fused):
    g = lstm_seq.load(golden_dir)
    c = g["cases"][case]
    m = lstm_seq.model_for(g, case, fused=fused)
    out, cost, _, _ = lstm_seq.run_case(m, g, case, golden_dir)
    cost.backward()
    assert torch.allclose(out, c["out"], rtol=1e-4, atol=1e-5), float((out - c["out"]).abs().max())
    assert torch.allclose(cost, c["loss"], rtol=1e-4, atol=1e-6)
    _check_grads(m, c)
    S = out.shape[0]
    # the parameters are fixed, so the pack runs once; the first step has H = C = None, every later one carries them
    assert dense_rows == (["pack"] + ["fwd"] * S + ["bwd", "wgrad"] * S if fused else [])


def test_weight_pack_is_the_gate_weights_in_basis_order(dense_rows):
    torch.manual_seed(0)
    for K, cin, bias in ((2, 14, True), (1, 16, True), (2, 3, False)):
        m = GConvLSTM(cin, 32, K, bias=bias)
        w, b, peep = m._rows_packed()
        assert w.shape == (128, K * (cin + 32)) and torch.equal(w, m._weight().t())
        want = torch.cat([getattr(m, f"b_{g}").reshape(32) for g in "ifco"])
        if bias:
            want = m._conv_bias() + want
        assert torch.allclose(b, want) and torch.equal(peep, torch.cat([m.w_c_i, m.w_c_f, m.w_c_o]))
        assert m._rows_packed()[0] is w                               # cached until a parameter changes
        with torch.no_grad():
            m.conv_x_i.lins[0].weight.add_(1.0)
        assert m._rows_packed()[0] is not w
        g = GCLSTM(cin, 32, K, bias=bias)
        w, b = g._rows_packed()
        assert w.shape == (128, cin + 32 * K) and torch.equal(w, g._weight().t())
        assert torch.allclose(b, torch.cat(g._gate_bias()))


@pytest.mark.parametrize("module", ["gconvlstm", "gclstm"])
def test_state_gradients_with_either_output_gradient_absent(golden_dir, dense_rows, module):
    """dX, dH, dC and every parameter gradient equal autograd's when the loss reads H' only, C' only or both (gH or gC is None), with
    H and C given or None; a None state has no gradient and leaves the structurally zero parameter gradients exactly zero."""
    ei, ew, X, _, _, _ = lstm_seq.data("chickenpox", golden_dir)
    torch.manual_seed(3)
    cls = lstm_seq.MODULES[module]
    fused, ref = cls(4, 32, 2), cls(4, 32, 2)
    with torch.no_grad():
        for p in fused.parameters():
            p.add_(torch.randn_like(p) * 0.1)
    ref.load_state_dict(fused.state_dict())
    ref.fused_training = False
    H, C = torch.randn(20, 32) * 0.5, torch.randn(20, 32)
    wh, wc = torch.randn(20, 32), torch.randn(20, 32)
    for use in ("h", "c", "hc"):
        for with_state in (True, False):
            res = []
            for m in (fused, ref):
                m.zero_grad(set_to_none=True)
                x = X[5].clone().requires_grad_(True)
                h = H.clone().requires_grad_(True) if with_state else None
                c = C.clone().requires_grad_(True) if with_state else None
                hn, cn = m(x, ei, ew, h, c)
                if use == "h":
                    loss = (hn * wh).sum()
                elif use == "c":
                    loss = (cn * wc).sum()
                else:
                    loss = (hn * wh).sum() + (cn * wc).sum()
                loss.backward()
                res.append((hn.detach(), cn.detach(), x.grad, None if h is None else h.grad, None if c is None else c.grad,
                            {k: p.grad for k, p in m.named_parameters()}))
            (hf, cf, *gf, pf), (ha, ca, *ga, pa) = res
            assert torch.allclose(hf, ha, rtol=1e-5, atol=1e-6) and torch.allclose(cf, ca, rtol=1e-5, atol=1e-6)
            for a, b in zip(gf, ga):
                assert (a is None) == (b is None)
                if b is not None:
                    assert torch.allclose(a, b, rtol=1e-4, atol=1e-6)
            for k in pa:
                if pa[k] is None:                                     # autograd leaves an unused parameter without a gradient
                    assert pf[k] is None or torch.all(pf[k] == 0), k
                else:
                    assert torch.allclose(pf[k], pa[k], rtol=1e-4, atol=1e-6), k
            if not with_state:
                for k, v in pf.items():
                    h_weight = k.startswith("conv_h_") if module == "gconvlstm" else k.startswith("conv_")
                    if h_weight and ".lins." in k:
                        assert torch.all(v == 0), k                   # H = None: the H columns of the basis are zero
                    if k in ("w_c_i", "w_c_f"):
                        assert torch.all(v == 0), k                   # C = None: dpi * C and dpf * C vanish


def test_gradient_blocks_and_bias_copies_do_not_alias(golden_dir, dense_rows):
    """Every bias of a gate receives the gate's bias gradient as a separate tensor, and a second backward accumulates into each .grad on
    its own."""
    g = lstm_seq.load(golden_dir)
    for case in ("gconvlstm_chickenpox_K2_sym", "gclstm_chickenpox_K2_sym"):
        c = g["cases"][case]
        m = lstm_seq.model_for(g, case)
        for _ in range(2):
            lstm_seq.run_case(m, g, case, golden_dir)[1].backward()
        r = m.recurrent
        ptrs = [p.grad.data_ptr() for p in r.parameters()]
        assert len(set(ptrs)) == len(ptrs) or isinstance(r, GConvLSTM)   # GConvLSTM's weight blocks are views of one dw
        for gate in "ifco":
            bs = [getattr(r, f"b_{gate}")] + ([getattr(r, f"conv_x_{gate}").bias, getattr(r, f"conv_h_{gate}").bias] if isinstance(r, GConvLSTM)
                                              else [getattr(r, f"conv_{gate}").bias])
            assert len({b.grad.data_ptr() for b in bs}) == len(bs)
            key = f"recurrent.b_{gate}"
            assert torch.allclose(bs[0].grad, 2 * c["grads"][key], rtol=1e-3, atol=1e-6)
            for b in bs[1:]:
                assert torch.allclose(b.grad.reshape(-1), bs[0].grad.reshape(-1))


def test_routing(golden_dir, dense_rows, monkeypatch):
    ei, ew, X, _, _, _ = lstm_seq.data("chickenpox", golden_dir)
    x = X[0]
    H = torch.randn(20, 32) * 0.5
    # outside the envelope: op-for-op, with gradients (GConvLSTM in 17 falls to its autograd path: (K * Cw) % 64 != 0)
    for cls in (GConvLSTM, GCLSTM):
        for m, xx, h in ((cls(17, 32, 2), torch.randn(20, 17), H), (cls(4, 32, 3), x, H), (cls(4, 16, 2), x, H[:, :16]),
                         (cls(4, 32, 2), x.expand(2, 20, 4), H.expand(2, 20, 32))):
            hn, cn = m(xx, ei, ew, h)
            (hn.sum() + cn.sum()).backward()
            assert all(p.grad is not None for p in m.parameters())
    assert dense_rows == []
    for cls in (GConvLSTM, GCLSTM):
        m = cls(4, 32, 2)
        m.fused_training = False                                      # training calls stay op-for-op ...
        sum(t.sum() for t in m(x, ei, ew, H)).backward()
        assert dense_rows == []
        with torch.no_grad():                                         # ... inference does not depend on the switch
            m(x, ei, ew, H)
        assert dense_rows == ["pack", "fwd"]
        dense_rows.clear()
    # out = 16 cells never consult the library (their inference runs other kernels, so only training calls are made here)
    monkeypatch.setattr(ops, "lstm_rows_supported", lambda *a, **k: pytest.fail("row-split entry consulted"))
    for cls in (GConvLSTM, GCLSTM):
        m = cls(4, 16, 2)
        sum(t.sum() for t in m(x, ei, ew)).backward()
        sum(t.sum() for t in m(x, ei, ew, H[:, :16], H[:, 16:])).backward()
    assert dense_rows == []
