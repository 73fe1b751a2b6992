"""Host-side logic of the ChebConv-family modules (weight folding, gate order, shared Chebyshev basis, timestep folding,
the MSTGCN reshape, autograd through the torch part) checked on the CPU against the committed reference goldens.  The
two things that need a GPU -- the cached plan and `stmp_spmm` -- are replaced by a dense Laplacian built with the oracle's
`cheb_norm`; the modules run their autograd (training) code path, which is plain torch around those two calls.  For the Chebyshev
cells' `no_grad` routes the gate kernels (`stmp_gemm_lstm_f32`, `stmp_lstm_ifc` / `_oh`, `stmp_gru_zr` / `_out`) are replaced too, by
stand-ins that hold every operand to the element count the kernel indexes."""
import os

import pytest
import torch

from oracle import pyg
from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.attention import MSTGCN, STConv
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvGRU, GConvLSTM
import pytorch_geometric_temporal_b200.nn.recurrent._cheb as cheb_mod
import pytorch_geometric_temporal_b200.nn.recurrent.gc_lstm as gc_mod
import pytorch_geometric_temporal_b200.nn.recurrent.gconv_gru as gru_mod
import pytorch_geometric_temporal_b200.nn.recurrent.gconv_lstm as lstm_mod


class _DensePlan(object):
    def __init__(self, L):
        self.L = L


@pytest.fixture()
def dense_graph_ops(monkeypatch):
    def plan(self, edge_index, edge_weight, num_nodes, normalization, lambda_max, batch=None):
        lam = self._lambda_value(lambda_max)
        e, w = pyg.cheb_norm(edge_index, num_nodes, edge_weight, normalization, lam)
        L = torch.zeros(num_nodes, num_nodes)
        L.index_put_((e[1], e[0]), w, accumulate=True)              # out[dst] += w * x[src]
        return _DensePlan(L)

    def spmm(plan, op, x, alpha=1.0, z=None, beta=0.0, att=None):
        y = alpha * torch.matmul(plan.L, x)
        return y if z is None else y + beta * z

    def spmm_cols(plan, op, buf, src, dst, width, alpha=1.0, z_col=None, beta=0.0, transposed=False):
        y = alpha * torch.matmul(plan.L, buf[..., src:src + width])
        buf[..., dst:dst + width] = y if z_col is None else y + beta * buf[..., z_col:z_col + width]

    # The kernels of the `no_grad` routes index flat buffers with one row count for every operand; the stand-ins hold each operand to
    # exactly the elements the kernel would read or write, and compute on those flat rows.
    def counts(n, *ts):
        assert all(t.numel() == n for t in ts), (n, [t.numel() for t in ts])

    def lstm_chain(pre, cell, cout, cb, wci, wcf, wco, bi, bf, bc, bo):
        v = lambda t: t.reshape(-1)
        pre = pre if cb is None else pre + v(cb)
        pi, pf, pc, po = (pre[:, j * cout:(j + 1) * cout] for j in range(4))
        cn = torch.sigmoid(pf + v(wcf) * cell + v(bf)) * cell + torch.sigmoid(pi + v(wci) * cell + v(bi)) * torch.tanh(pc + v(bc))
        return torch.sigmoid(po + v(wco) * cn + v(bo)) * torch.tanh(cn), cn

    def gemm_lstm(A, packed, K, cout, cb, cell, wci, wcf, wco, bi, bf, bc, bo):
        M = A.numel() // K                                          # stmp_gemm_lstm_f32: one cell row per row of A
        counts(M * K, A)
        counts(M * cout, cell)
        counts(cout, wci, wcf, wco, bi, bf, bc, bo)
        h, c = lstm_chain(A.reshape(M, K) @ packed, cell.reshape(M, cout), cout, cb, wci, wcf, wco, bi, bf, bc, bo)
        return h.view(cell.shape), c.view(cell.shape)

    def lstm_ifc(pi, pf, pc, c, wci, wcf, bi, bf, bc):
        cout = pi.size(-1)
        counts(pi.numel(), pf, pc, c)
        counts(cout, wci, wcf, bi, bf, bc)
        flat = [t.reshape(-1, cout) for t in (pi, pf, pc)]
        pre = torch.cat(flat + [torch.zeros_like(flat[0])], dim=1)
        zero = torch.zeros(cout)
        return lstm_chain(pre, c.reshape(-1, cout), cout, None, wci, wcf, zero, bi, bf, bc, zero)[1].view(pi.shape)

    def lstm_oh(po, cnew, wco, bo):
        cout = po.size(-1)
        counts(po.numel(), cnew)
        counts(cout, wco, bo)
        cn = cnew.reshape(-1, cout)
        return (torch.sigmoid(po.reshape(-1, cout) + wco.reshape(-1) * cn + bo.reshape(-1)) * torch.tanh(cn)).view(po.shape)

    def gru_zr(pz, pr, h):
        counts(pz.numel(), pr, h)
        z, r = torch.sigmoid(pz), torch.sigmoid(pr)
        return z, r, h.reshape(pz.shape) * r

    def gru_out(ph, z, h):
        counts(ph.numel(), z, h)
        return z * h.reshape(ph.shape) + (1 - z) * torch.tanh(ph)

    monkeypatch.setattr(cheb_mod.ChebPlanMixin, "_cheb_plan", plan)
    for name, fn in dict(spmm=spmm, spmm_cols=spmm_cols, gemm_prepack=lambda W: W.clone(), gemm_lstm=gemm_lstm, lstm_ifc=lstm_ifc,
                         lstm_oh=lstm_oh, gru_zr=gru_zr, gru_out=gru_out).items():
        monkeypatch.setattr(ops, name, fn)
    for m in (gc_mod, gru_mod, lstm_mod):
        monkeypatch.setattr(m, "_require_cuda", lambda *a, **k: None)
    monkeypatch.setattr(GConvGRU, "_fused_ok", lambda self, plan, X, H: False)


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


def _loss(outs):
    return sum((o * torch.linspace(-1, 1, o.numel()).view_as(o)).sum() for o in outs)


def _close(a, b, rtol=1e-4, atol=1e-5):
    assert a.shape == b.shape and torch.allclose(a, b, rtol=rtol, atol=atol), float((a - b).abs().max())


def test_gconv_gru_and_lstm_host_logic(golden_dir, dense_graph_ops):
    g = _load(golden_dir, "gconv_gru_small")
    for c in g["cases"].values():
        m = GConvGRU(4, 16, c["K"], normalization=c["normalization"])
        m.load_state_dict(c["state"])
        _close(m(c["X"], g["edge_index"], g["edge_weight"], c["H"], c["lambda_max"]), c["out"])
    g = _load(golden_dir, "gconv_lstm_small")
    for c in g["cases"].values():
        m = GConvLSTM(4, 16, c["K"])
        m.load_state_dict(c["state"])
        h, cc = m(c["X"], g["edge_index"], g["edge_weight"], c["H"], c["C"])
        _close(h, c["outH"]); _close(cc, c["outC"])
        h, cc = m(c["X"], g["edge_index"])
        _close(h, c["outH0"]); _close(cc, c["outC0"])


def test_gc_lstm_host_logic_with_gradients(golden_dir, dense_graph_ops):
    g = _load(golden_dir, "gc_lstm_small")
    for name, c in g["cases"].items():
        if "grads" not in c:
            continue
        m = GCLSTM(4, 16, c["K"], normalization=c["normalization"])
        m.load_state_dict(c["state"])
        x, h, cc = (t.clone().requires_grad_(True) for t in (c["X"], c["H"], c["C"]))
        ho, co = m(x, g["edge_index"], g["edge_weight"], h, cc, c["lambda_max"])
        _close(ho, c["outH"]); _close(co, c["outC"])
        _loss([ho, co]).backward()
        for k, p in m.named_parameters():
            _close(p.grad, c["grads"][k], 1e-3, 1e-5)
        _close(x.grad, c["gX"], 1e-3, 1e-5); _close(h.grad, c["gH"], 1e-3, 1e-5); _close(cc.grad, c["gC"], 1e-3, 1e-5)


def test_no_grad_routes_host_logic(golden_dir, dense_graph_ops):
    """The `no_grad` routes of the three cells -- the pointwise gate kernels, and GCLSTM's fused GEMM at 32 channels -- against the same
    goldens."""
    with torch.no_grad():
        g = _load(golden_dir, "gconv_gru_small")
        for c in g["cases"].values():
            m = GConvGRU(4, 16, c["K"], normalization=c["normalization"])
            m.load_state_dict(c["state"])
            _close(m(c["X"], g["edge_index"], g["edge_weight"], c["H"], c["lambda_max"]), c["out"])
        g = _load(golden_dir, "gconv_lstm_small")
        for c in g["cases"].values():
            m = GConvLSTM(4, 16, c["K"])
            m.load_state_dict(c["state"])
            h, cc = m(c["X"], g["edge_index"], g["edge_weight"], c["H"], c["C"])
            _close(h, c["outH"]); _close(cc, c["outC"])
        g = _load(golden_dir, "gc_lstm_small")
        for c in g["cases"].values():                               # (4, 16, K) on the pointwise kernels, (8, 32, 3) on the fused GEMM
            m = GCLSTM(*c["state"]["W_i"].shape, c["K"], normalization=c["normalization"])
            m.load_state_dict(c["state"])
            h, cc = m(c["X"], g["edge_index"], g["edge_weight"], c["H"], c["C"], c["lambda_max"])
            _close(h, c["outH"]); _close(cc, c["outC"])


def _oracle_cell(name, p, X, ei, ew, state):
    return {"gconv_gru": lambda: [R.gconv_gru_cell(p, X, ei, ew, *state)], "gconv_lstm": lambda: list(R.gconv_lstm_cell(p, X, ei, ew, *state)),
            "gc_lstm": lambda: list(R.gc_lstm_cell(p, X, ei, ew, *state))}[name]()


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("cin,cout,K", [(4, 16, 3), (8, 32, 3)])
@pytest.mark.parametrize("name", ["gconv_gru", "gconv_lstm", "gc_lstm"])
def test_state_shared_across_a_batch_matches_reference(dense_graph_ops, name, cin, cout, K, train):
    """X (B, N, F) with H (and C) of (N, out): the reference broadcasts the state over the batch (its elementwise sums of the convolutions
    and w_c * C), and its gradient sums over the windows.  `no_grad` runs the fused GEMM + gate epilogue at 32 channels and the pointwise
    gate kernels at 16; with gradients, the op-for-op path (GConvLSTM's `_LstmCellFn` is pinned in test_gconv_lstm_backward_algebra_cpu)."""
    B, n = 3, 24
    torch.manual_seed(cin + cout)
    ei = torch.stack([torch.randint(0, n, (90,)), torch.randint(0, n, (90,))])
    ei = torch.unique(ei[:, ei[0] != ei[1]], dim=1)
    ew = torch.rand(ei.size(1)) + 0.1
    m = {"gconv_gru": GConvGRU, "gconv_lstm": GConvLSTM, "gc_lstm": GCLSTM}[name](cin, cout, K)
    m.fused_training = False
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("bias") or k.startswith("b_"):
                p.normal_(0, 0.2)
    ns = 1 if name == "gconv_gru" else 2
    X, S = torch.randn(B, n, cin), [0.5 * torch.randn(n, cout) for _ in range(ns)]
    wgts = [torch.randn(B, n, cout) for _ in range(ns)]
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    ref_leaves = [t.clone().requires_grad_(True) for t in [X] + S]
    ref = _oracle_cell(name, p, ref_leaves[0], ei, ew, ref_leaves[1:])
    assert all(r.shape == (B, n, cout) for r in ref)
    sum((r * w).sum() for r, w in zip(ref, wgts)).backward()
    leaves = [t.clone().requires_grad_(train) for t in [X] + S]
    with torch.set_grad_enabled(train):
        out = m(leaves[0], ei, ew, *leaves[1:])
    out = [out] if name == "gconv_gru" else list(out)
    for o, r in zip(out, ref):
        _close(o, r.detach(), 1e-5, 1e-6)
    if not train:
        return
    sum((o * w).sum() for o, w in zip(out, wgts)).backward()
    for label, a, b in zip(["dX", "dH", "dC"], leaves, ref_leaves):
        assert a.grad.shape == b.grad.shape, label
        _close(a.grad, b.grad, 1e-4, 1e-5)
    for k, q in m.named_parameters():
        _close(q.grad, p[k].grad, 1e-4, 1e-4 * float(p[k].grad.abs().max()) + 1e-6)


def test_cell_operand_guards_reject_what_the_kernel_would_overrun():
    """`ops` checks every operand of the pointwise and epilogue kernels against the rows the kernel walks before it touches the device:
    a state of N rows beside gates of B N rows is refused, as is a per-channel vector of the wrong width."""
    rows, Co = 6, 4
    g, st, v = torch.zeros(rows, Co), torch.zeros(rows // 2, Co), torch.zeros(Co)
    bad = [lambda: ops.lstm_ifc(g, g, g, st, v, v, v, v, v), lambda: ops.lstm_ifc(g, g, g, g, v, torch.zeros(Co + 1), v, v, v),
           lambda: ops.lstm_oh(g, st, v, v), lambda: ops.lstm_oh(g, g, v, torch.zeros(1)), lambda: ops.gru_zr(g, g, st),
           lambda: ops.gru_out(g, st, g), lambda: ops.gru_out(g, g, st),
           lambda: ops.lstm_gate_bwd(torch.zeros(rows, 4 * Co), g, st, None, None, *[v] * 7),
           lambda: ops.lstm_gate_bwd(torch.zeros(rows // 2, 4 * Co), g, g, None, None, *[v] * 7),
           lambda: ops.lstm_gate_bwd(torch.zeros(rows, 4 * Co), g, g, g, st, *[v] * 7),
           lambda: ops.gemm_lstm(torch.zeros(rows, 8), None, 8, Co, None, st, *[v] * 7),
           lambda: ops.gemm_lstm(torch.zeros(rows, 8), None, 8, Co, v, g, *[v] * 7),
           lambda: ops.gemm_lstm(torch.zeros(rows, 8), None, 8, Co, None, g, *[v] * 6, torch.zeros(2 * Co))]
    for i, call in enumerate(bad):
        with pytest.raises(RuntimeError, match="elements, the kernel indexes"):
            call()
    # operands of the right sizes pass the guard and reach the device check (CPU tensors here)
    for call in (lambda: ops.lstm_ifc(g, g, g, g, *[v] * 5), lambda: ops.gru_out(g, g, g),
                 lambda: ops.gemm_lstm(torch.zeros(rows, 8), None, 8, Co, torch.zeros(4 * Co), g, *[v] * 7)):
        with pytest.raises(RuntimeError, match="CUDA only"):
            call()


def test_stconv_host_logic_with_gradients(golden_dir, dense_graph_ops):
    g = _load(golden_dir, "stconv_small")
    for name, c in g["cases"].items():
        m = STConv(K=c["K"], normalization=c["normalization"], **g["ctor"])
        m.load_state_dict(c["state"])
        m.eval()
        with torch.no_grad():
            _close(m(c["X"], g["edge_index"], g["edge_weight"]), c["out_eval"])
            _close(m(c["X"], g["edge_index"]), c["out_eval_noew"])
        m.train()
        X = c["X"].clone().requires_grad_(True)
        out = m(X, g["edge_index"], g["edge_weight"])
        _close(out, c["out_train"])
        _loss([out]).backward()
        for k, p in m.named_parameters():                         # BatchNorm backward: bar relative to the tensor's max
            _close(p.grad, c["grads"][k], 0.0, 2e-4 * float(c["grads"][k].abs().max()) + 1e-6)
        _close(X.grad, c["gX"], 0.0, 2e-4 * float(c["gX"].abs().max()) + 1e-6)


def test_mstgcn_host_logic_with_gradients(golden_dir, dense_graph_ops):
    g = _load(golden_dir, "mstgcn_small")
    for name, c in g["cases"].items():
        m = MSTGCN(time_strides=c["time_strides"], **g["ctor"])
        m.load_state_dict(c["state"])
        X = c["X"].clone().requires_grad_(True)
        out = m(X, g["edge_index"])
        _close(out, c["out"], 2e-4, 2e-5)
        _loss([out]).backward()
        for k, p in m.named_parameters():
            _close(p.grad, c["grads"][k], 2e-3, 2e-5)
        _close(X.grad, c["gX"], 2e-3, 2e-5)
        with torch.no_grad():
            _close(m(c["X"], [g["edge_index"]] * 6), c["out_list"], 2e-4, 2e-5)


# ---- DConv / DCRNN (tiled path) and the GCNConv family ------------------------------------------------------------------
import pytorch_geometric_temporal_b200.nn.recurrent.attentiontemporalgcn as a3_mod  # noqa: E402
import pytorch_geometric_temporal_b200.nn.recurrent.dcrnn as dcrnn_mod  # noqa: E402
import pytorch_geometric_temporal_b200.nn.recurrent.temporalgcn as tgcn_mod  # noqa: E402
from oracle import recurrent as R  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN, A3TGCN2, DCRNN, BatchedDCRNN, TGCN, TGCN2  # noqa: E402


class _DensePair(object):
    def __init__(self, mats):
        self.mats = mats


def _dense(edge_index, w, n):
    M = torch.zeros(n, n)
    M.index_put_((edge_index[1], edge_index[0]), w, accumulate=True)
    return M


@pytest.fixture()
def dense_dconv_gcn_ops(monkeypatch):
    def dconv_plan(self, edge_index, edge_weight, num_nodes):
        ew = edge_weight if edge_weight is not None else torch.ones(edge_index.size(1))
        eo, no, ei, ni = R.dconv_operators(edge_index, ew, self._batched_semantics, num_nodes)
        return _DensePair([_dense(eo, no, num_nodes), _dense(ei, ni, num_nodes)])

    def gcn_plan(self, edge_index, edge_weight, num_nodes):
        e, w = pyg.gcn_norm(edge_index, edge_weight, num_nodes, self.improved, self.add_self_loops, torch.float32)
        return _DensePair([_dense(e, w, num_nodes)])

    def spmm(plan, op, x, alpha=1.0, z=None, beta=0.0, att=None):
        y = alpha * torch.matmul(plan.mats[op], x)
        return y if z is None else y + beta * z

    monkeypatch.setattr(dcrnn_mod.DConv, "_plan", dconv_plan)
    monkeypatch.setattr(dcrnn_mod.DCRNN, "_plan", dconv_plan)
    monkeypatch.setattr(tgcn_mod.TGCN, "_plan", gcn_plan)
    monkeypatch.setattr(ops, "spmm", spmm)
    monkeypatch.setattr(ops, "dcrnn_seq_supported", lambda *a, **k: False)          # no fused kernels on the CPU
    monkeypatch.setattr(tgcn_mod.TGCN, "_fused_ok", lambda self, plan, X, H: False)
    for m in (dcrnn_mod, tgcn_mod, a3_mod):
        monkeypatch.setattr(m, "_require_cuda", lambda *a, **k: None)


def test_dcrnn_tiled_host_logic_with_gradients(golden_dir, dense_dconv_gcn_ops):
    for K in (1, 3, 4):
        g = _load(golden_dir, f"dcrnn_small_K{K}")
        m = DCRNN(3, 16, K)
        m.load_state_dict(g["state"])
        x, h = g["X"].clone().requires_grad_(True), g["H"].clone().requires_grad_(True)
        out = m(x, g["edge_index"], g["edge_weight"], h)
        _close(out, g["out"])
        _loss([out]).backward()
        for k, p in m.named_parameters():
            _close(p.grad, g["grads"][k], 1e-3, 1e-5)
        _close(x.grad, g["gX"], 1e-3, 1e-5); _close(h.grad, g["gH"], 1e-3, 1e-5)
    g = _load(golden_dir, "dcrnn_small_batched_K3")
    m = BatchedDCRNN(3, 16, 3)
    m.load_state_dict(g["state"])
    _close(m(g["X"], g["edge_index"], g["edge_weight"]), g["out"])
    g = _load(golden_dir, "dcrnn_cfg2_cell")
    m = DCRNN(2, 32, 2)
    m.load_state_dict(g["state"])
    _close(m(g["X"], g["edge_index"], g["edge_weight"], g["H"]), g["out"])
    _close(m(g["X"], g["edge_index"]), g["out_noew_noh"])                      # edge_weight None, H None


def test_tgcn_family_host_logic(golden_dir, dense_dconv_gcn_ops):
    g = _load(golden_dir, "tgcn_small")
    for c in g["cases"].values():
        m = TGCN(4, 16, improved=c["improved"], add_self_loops=c["add_self_loops"])
        m.load_state_dict(c["state"])
        _close(m(c["X"], g["edge_index"], g["edge_weight"], c["H"]), c["out"])
        m2 = TGCN2(4, 16, 3, improved=c["improved"], add_self_loops=c["add_self_loops"])
        m2.load_state_dict(c["state2"])
        _close(m2(c["X2"], g["edge_index"], g["edge_weight"], c["H2"]), c["out2"])
    g = _load(golden_dir, "a3tgcn_small")
    m = A3TGCN2(2, 16, 6, 3)
    m.load_state_dict(g["state"])
    _close(m(g["X"], g["edge_index"], g["edge_weight"]), g["out"])
    _close(m(g["X"], g["edge_index"], g["edge_weight"], torch.ones(3, 40, 16) * 0.3), g["outH"])
    m1 = A3TGCN(2, 16, 6)
    m1.load_state_dict(g["state1"])
    _close(m1(g["X1"], g["edge_index"], g["edge_weight"]), g["out1"])


def test_tgcn_attention_folding_host_logic_vs_reference_golden(golden_dir, dense_dconv_gcn_ops, monkeypatch):
    """Host side of the fused temporal-attention + GCN kernel (stmp_tgcn_attn_fwd): the folded weights (A, Bm, c) of
    `TGCN._packed3`, the period softmax and the call shapes, with the kernel replaced by a dense restatement of its
    arithmetic -- against the UNMODIFIED reference modules at the PEMS-BAY shape (325 nodes)."""
    def fake_kernel(plan, x, A, Bm, c, probs=None, h=None, h_shared=False):
        B, N, Fi, P = x.shape
        L = plan.mats[0]
        H = torch.zeros(B, N, 32) if h is None else (h.expand(B, N, 32) if h_shared else h.reshape(B, N, 32))
        out = torch.zeros(B, N, 32)
        for t in range(P):
            ax = torch.matmul(L, x[..., t])                                     # (B,N,Fi): A^ X_t
            pre = lambda g, Hp: ax @ A[:, 32 * g:32 * g + 32] + Hp @ Bm[:, 32 * g:32 * g + 32] + c[32 * g:32 * g + 32]
            Z, Rg = torch.sigmoid(pre(0, H)), torch.sigmoid(pre(1, H))
            Hn = Z * H + (1 - Z) * torch.tanh(pre(2, H * Rg))
            out = out + (Hn if probs is None else probs[t] * Hn)
        return out
    monkeypatch.setattr(ops, "tgcn_attn_fwd", fake_kernel)
    g = _load(golden_dir, "a3tgcn2_cfg3")
    ei, ew, X, H = g["edge_index"], g["edge_weight"], g["X"], g["H"]
    with torch.no_grad():
        m = A3TGCN2(2, 32, 12, 64)
        m.load_state_dict(g["state"])
        _close(m(X, ei, ew), g["out"]); _close(m(X, ei, ew, H), g["outH"])
        m1 = A3TGCN(2, 32, 12)
        m1.load_state_dict(g["state1"])
        _close(m1(X[0], ei, ew), g["out1"]); _close(m1(X[0], ei, ew, H[0]), g["out1H"])
        c2 = TGCN2(2, 32, 8)
        c2.load_state_dict(g["state_cell"])
        _close(c2(X[..., 0], ei, ew), g["cell"]); _close(c2(X[..., 0], ei, ew, H), g["cellH"])


def test_tgcn_attention_training_host_logic_vs_reference_golden_gradients(golden_dir, dense_dconv_gcn_ops, monkeypatch):
    """Host side of the fused TRAINING path (stmp_tgcn_attn_fwd + stmp_tgcn_attn_bwd): the differentiable folding `TGCN._fold3`, the
    softmax of the attention and the routing (no state, no input gradient -> `ops.tgcn_attn_train`), with the kernel pair replaced by a
    dense differentiable restatement -- output and EVERY parameter gradient against the unmodified reference at the PEMS-BAY shape."""
    calls = []

    def fake_train(plan, x, A, Bm, c, probs=None):
        calls.append(tuple(x.shape))
        L = plan.mats[0]
        out = 0
        for t in range(x.shape[-1]):
            ax = torch.matmul(L, x[..., t])
            Z = torch.sigmoid(ax @ A[:, 0:32] + c[0:32])
            Ht = torch.tanh(ax @ A[:, 64:96] + c[64:96])                       # H = 0: the r gate and Bm drop out
            out = out + (1 - Z) * Ht * (1.0 if probs is None else probs[t])
        return out
    monkeypatch.setattr(ops, "tgcn_attn_train", fake_train)
    g = _load(golden_dir, "a3tgcn2_cfg3_grads")
    ei, ew, X = g["edge_index"], g["edge_weight"], g["X"]
    m = A3TGCN2(2, 32, 12, 8)
    m.load_state_dict(g["state"])
    out = m(X, ei, ew)
    w = torch.linspace(-1, 1, out.numel()).view_as(out)
    (out * w).sum().backward()
    _close(out, g["out"])
    for k, p in m.named_parameters():
        ref = g["grads"][k]
        assert p.grad is not None, k
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-6), k
    c2 = TGCN2(2, 32, 8)
    c2.load_state_dict(g["state_cell"])
    cell = c2(X[..., 3], ei, ew)
    (cell * w).sum().backward()
    _close(cell, g["cell"])
    for k, p in c2.named_parameters():
        ref = g["grads_cell"][k]
        assert torch.allclose(p.grad, ref, rtol=1e-3, atol=1e-3 * float(ref.abs().max()) + 1e-6), k
    assert calls == [(8, 325, 2, 12), (8, 325, 2, 1)]
    # a call with an incoming state stays on the op-for-op path
    m(X[:2], ei, ew, torch.zeros(2, 325, 32)).sum().backward()
    assert len(calls) == 2


# ---- ASTGCN: attention-weighted first hop, timesteps folded into the feature axis, fp32 time convolutions ---------------
import pytorch_geometric_temporal_b200.nn.attention.astgcn as astgcn_mod  # noqa: E402
from oracle import attention as OA  # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN  # noqa: E402


@pytest.fixture()
def dense_att_ops(monkeypatch):
    def plan(self, edge_index, edge_weight, num_nodes, lambda_max, batch=None):
        lam = torch.tensor(2.0 if lambda_max is None else float(lambda_max))
        ei, w = OA.cheb_att_norm(edge_index, num_nodes, edge_weight, self._normalization, lam)
        W = torch.zeros(num_nodes, num_nodes)
        W.index_put_((ei[0], ei[1]), w, accumulate=True)          # propagated on the TRANSPOSED index: out[row] += w x[col]
        return _DensePlan(W)

    def spmm(plan, op, x, alpha=1.0, z=None, beta=0.0, att=None):
        A = plan.L if att is None else plan.L.unsqueeze(0) * att  # first hop: norm * S[b,row,col]
        y = alpha * torch.matmul(A, x)
        return y if z is None else y + beta * z

    monkeypatch.setattr(astgcn_mod.ChebConvAttention, "_plan", plan)
    monkeypatch.setattr(ops, "spmm", spmm)
    monkeypatch.setattr(astgcn_mod, "_require_cuda", lambda *a, **k: None)


def test_astgcn_host_logic(golden_dir, dense_att_ops):
    g = _load(golden_dir, "astgcn_small")
    for name, c in g["cases"].items():
        m = ASTGCN(**g["ctor"], normalization=c["normalization"])
        m.load_state_dict(c["state"])
        X = c["X"].clone().requires_grad_(True)
        out = m(X, g["edge_index"])
        _close(out, c["out"], 2e-4, 2e-5)
        out.sum().backward()                                      # the whole block is differentiable through the stand-ins
        assert torch.isfinite(X.grad).all() and all(torch.isfinite(p.grad).all() for p in m.parameters())
        with torch.no_grad():
            _close(m(c["X"], [g["edge_index"]] * 6), c["out"], 2e-4, 2e-5)      # per-timestep list of the same graph
