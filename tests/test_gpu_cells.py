"""GPU parity of the ChebConv / GCNConv cells and ASTGCN through the public modules, against the committed
reference goldens (tests/golden/make_goldens.py).  Strict fp32: rtol=1e-4, atol=1e-5."""
import os

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.dataset import ChickenpoxDatasetLoader, synthetic
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN, ChebConvAttention
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN, A3TGCN2, GConvGRU, GConvLSTM, TGCN, TGCN2

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got = got.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def test_gconv_gru_goldens(golden_dir):
    g = _load(golden_dir, "gconv_gru_small")
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    for name, c in g["cases"].items():
        m = GConvGRU(4, 16, c["K"], normalization=c["normalization"]).to(DEV)
        m.load_state_dict(c["state"])
        lm = None if c["lambda_max"] is None else c["lambda_max"].to(DEV)
        n0 = _lib.launch_count()
        with torch.no_grad():
            _close(m(c["X"].to(DEV), ei, ew, c["H"].to(DEV), lm), c["out"])     # fused gate kernels
        assert c["K"] == 1 or _lib.launch_count() > n0
        _close(m(c["X"].to(DEV), ei, ew, c["H"].to(DEV), lm), c["out"])         # autograd path


def test_gconv_lstm_goldens(golden_dir):
    g = _load(golden_dir, "gconv_lstm_small")
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    for c in g["cases"].values():
        m = GConvLSTM(4, 16, c["K"]).to(DEV)
        m.load_state_dict(c["state"])
        with torch.no_grad():
            h, cc = m(c["X"].to(DEV), ei, ew, c["H"].to(DEV), c["C"].to(DEV))
            _close(h, c["outH"]); _close(cc, c["outC"])
            h, cc = m(c["X"].to(DEV), ei)                                         # no weights, no state
            _close(h, c["outH0"]); _close(cc, c["outC0"])
        h, cc = m(c["X"].to(DEV), ei, ew, c["H"].to(DEV), c["C"].to(DEV))        # autograd path
        _close(h, c["outH"]); _close(cc, c["outC"])


def test_gconv_gru_chickenpox_recurrence_config1():
    """BASELINE config 1: GConvGRU on the chickenpox signal (20 nodes, 4 lags), H carried over snapshots."""
    ds = ChickenpoxDatasetLoader().get_dataset(lags=4)
    torch.manual_seed(0)
    m = GConvGRU(4, 32, 2)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    mg = m.to(DEV)
    Hc, Hg = None, None
    for t, snap in enumerate(ds):
        if t == 12:
            break
        Hc = R.gconv_gru_cell(sd, snap.x, snap.edge_index, snap.edge_attr, Hc)
        s = snap.to(DEV)
        with torch.no_grad():
            Hg = mg(s.x, s.edge_index, s.edge_attr, Hg)
        _close(Hg, Hc)


def test_gconv_lstm_large_graph_vs_oracle():
    """cfg5 shape class: N=10^4, E=10^5, 64 hidden, K=3 (tiled path: SpMM kernels + cuBLAS)."""
    ei, ew = synthetic.large_graph(10000, 100000, 0)
    ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
    torch.manual_seed(0)
    m = GConvLSTM(64, 64, 3)
    X, H, C = torch.randn(10000, 64), torch.randn(10000, 64) * 0.5, torch.randn(10000, 64) * 0.5
    wh, wc = R.gconv_lstm_cell(m.state_dict(), X, ei, ew, H, C)
    with torch.no_grad():
        h, c = m.to(DEV)(X.to(DEV), ei.to(DEV), ew.to(DEV), H.to(DEV), C.to(DEV))
    _close(h, wh); _close(c, wc)


def test_tgcn_goldens(golden_dir):
    g = _load(golden_dir, "tgcn_small")
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    for c in g["cases"].values():
        m = TGCN(4, 16, improved=c["improved"], add_self_loops=c["add_self_loops"]).to(DEV)
        m.load_state_dict(c["state"])
        _close(m(c["X"].to(DEV), ei, ew, c["H"].to(DEV)), c["out"])
        m2 = TGCN2(4, 16, 3, improved=c["improved"], add_self_loops=c["add_self_loops"]).to(DEV)
        m2.load_state_dict(c["state2"])
        _close(m2(c["X2"].to(DEV), ei, ew, c["H2"].to(DEV)), c["out2"])


@pytest.mark.parametrize("fused", [True, False])
def test_gconv_lstm_cfg5_cell_sequence_gradients_vs_reference_golden(golden_dir, fused):
    """GConvLSTM(64,64,K=3) unrolled over 6 steps: final state AND every gradient against the UNMODIFIED reference's autograd
    (tests/golden/make_goldens_r2.py) -- through the hand-written cell backward (_LstmCellFn: wgmma GEMM + LSTM epilogue forward,
    recompute + stmp_lstm_gate_bwd + transposed SpMM backward) and through the op-for-op autograd path."""
    g = _load(golden_dir, "gconv_lstm_cfg5seq")
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    m = GConvLSTM(64, 64, 3).to(DEV)
    m.load_state_dict(g["state"])
    m.fused_training = fused
    X = g["X"].to(DEV).requires_grad_(True)
    c0 = _lib.path_counters()
    H = C = None
    loss = 0
    for t in range(6):
        H, C = m(X[t], ei, ew, H, C)
        loss = loss + (H * torch.linspace(-1, 1, H.numel(), device=DEV).view_as(H)).sum() + 0.3 * C.square().sum()
    loss.backward()
    assert (_ran(c0, "k_lstm_gate_bwd") == 6) == fused
    _close(H, g["H"]); _close(C, g["C"])
    _close(X.grad, g["gX"], 1e-3, 1e-3 * g["gX"].abs().max().item())
    for k, p in m.named_parameters():
        ref = g["grads"][k]
        _close(p.grad, ref, 1e-3, 1e-3 * ref.abs().max().item() + 1e-7)


def test_a3tgcn_goldens(golden_dir):
    g = _load(golden_dir, "a3tgcn_small")
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    m = A3TGCN2(2, 16, 6, 3).to(DEV)
    m.load_state_dict(g["state"])
    _close(m(g["X"].to(DEV), ei, ew), g["out"])
    _close(m(g["X"].to(DEV), ei, ew, torch.full((3, 40, 16), 0.3, device=DEV)), g["outH"])
    m1 = A3TGCN(2, 16, 6).to(DEV)
    m1.load_state_dict(g["state1"])
    _close(m1(g["X1"].to(DEV), ei, ew), g["out1"])


def _ran(before, name):
    return _lib.path_counters().get(name, 0) - before.get(name, 0)


def test_a3tgcn2_config3_shape_vs_oracle():
    """BASELINE config 3: A3TGCN2 on the PEMS-BAY shape (325 nodes, batch 64, 12 periods) through the fused
    temporal-attention + GCN kernel (stmp_tgcn_attn_fwd) -- ALL 64 rows against the oracle, with and without an incoming H."""
    ei, ew, _ = synthetic.pems_bay_like(0, 16)
    ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
    torch.manual_seed(0)
    m = A3TGCN2(2, 32, 12, 64)
    X = torch.randn(64, 325, 2, 12)
    H = torch.randn(64, 325, 32) * 0.5
    with torch.no_grad():
        want = R.a3tgcn(m.state_dict(), X, ei, ew)
        wantH = R.a3tgcn(m.state_dict(), X, ei, ew, H)
        md = m.to(DEV)
        c0 = _lib.path_counters()
        got = md(X.to(DEV), ei.to(DEV), ew.to(DEV))
        gotH = md(X.to(DEV), ei.to(DEV), ew.to(DEV), H.to(DEV))
    assert _ran(c0, "k_tgcn_attn") == 2 and _ran(c0, "k_spmm") == 0     # the fused kernel served both calls
    _close(got, want)
    _close(gotH, wantH)
    # training still goes through the differentiable tiled path and agrees with the fused inference result
    out_t = md(X[:4].to(DEV), ei.to(DEV), ew.to(DEV), H[:4].to(DEV))
    assert out_t.requires_grad
    _close(out_t, wantH[:4])


def test_a3tgcn_family_config3_vs_reference_golden(golden_dir):
    """The UNMODIFIED reference modules at the PEMS-BAY shape (tests/golden/make_goldens_r2.py): A3TGCN2, A3TGCN (one shared
    state) and a TGCN2 cell (the one-period case of the same kernel)."""
    from pytorch_geometric_temporal_b200.nn.recurrent import TGCN2
    g = _load(golden_dir, "a3tgcn2_cfg3")
    ei, ew, X, H = (g[k].to(DEV) for k in ("edge_index", "edge_weight", "X", "H"))
    c0 = _lib.path_counters()
    with torch.no_grad():
        m = A3TGCN2(2, 32, 12, 64).to(DEV)
        m.load_state_dict(g["state"])
        _close(m(X, ei, ew), g["out"])
        _close(m(X, ei, ew, H), g["outH"])
        m1 = A3TGCN(2, 32, 12).to(DEV)
        m1.load_state_dict(g["state1"])
        _close(m1(X[0], ei, ew), g["out1"])
        _close(m1(X[0], ei, ew, H[0]), g["out1H"])
        c2 = TGCN2(2, 32, 8).to(DEV)
        c2.load_state_dict(g["state_cell"])
        _close(c2(X[..., 0], ei, ew), g["cell"])
        _close(c2(X[..., 0], ei, ew, H), g["cellH"])
    assert _ran(c0, "k_tgcn_attn") == 6


def test_astgcn_goldens(golden_dir):
    g = _load(golden_dir, "astgcn_small")
    ei = g["edge_index"].to(DEV)
    for c in g["cases"].values():
        m = ASTGCN(**g["ctor"], normalization=c["normalization"]).to(DEV)
        m.load_state_dict(c["state"])
        n0 = _lib.launch_count()
        with torch.no_grad():
            out = m(c["X"].to(DEV), ei)
        assert _lib.launch_count() > n0
        _close(out, c["out"], rtol=2e-4, atol=2e-5)   # 2 blocks of softmax/LayerNorm amplify cuBLAS-vs-CPU GEMM rounding
        # per-timestep edge_index LIST path (astgcn.py:453-471)
        with torch.no_grad():
            out_l = m(c["X"].to(DEV), [ei] * c["X"].shape[-1])
        _close(out_l, c["out"], rtol=2e-4, atol=2e-5)


def test_astgcn_config4_shape_vs_reference_golden(golden_dir):
    """BASELINE configs[3] AT SHAPE: ASTGCN(3 blocks, K=3, 64/64 filters) on 307 nodes, batch 32 (and normalization None on 8
    rows), against the UNMODIFIED reference (tests/golden/make_goldens_r2.py) at the STRICT tolerance rtol 1e-4 / atol 1e-5,
    through the native channels-last path: fused spatial attention, blocked wgmma GEMMs (k_gemm_blocks), attention SpMM."""
    g = _load(golden_dir, "astgcn_cfg4")
    ei = g["edge_index"].to(DEV)
    for c in g["cases"].values():
        torch.manual_seed(c["seed"])                     # the reference module was built under this seed: same init stream
        m = ASTGCN(**g["ctor"], normalization=c["normalization"])
        chk = float(sum(v.double().abs().sum() for v in m.state_dict().values()))
        assert abs(chk - c["state_checksum"]) <= 1e-6 * c["state_checksum"], "parameter init stream differs from the reference module's"
        m = m.to(DEV)
        c0 = _lib.path_counters()
        with torch.no_grad():
            out = m(c["X"].to(DEV), ei)
        assert _ran(c0, "k_gemm_blocks") == 3 * 3 + 1       # per block: spatial attention, Chebyshev contraction, time conv; + final conv
        assert _ran(c0, "k_astgcn_factors") == 3
        assert _ran(c0, "k_spmm") == 6           # per block: attention-weighted hop + plain hop
        _close(out, c["out"])
        # the op-for-op torch path (what training uses) agrees as well
        out_t = m(c["X"][:4].to(DEV).requires_grad_(True), ei)
        _close(out_t, c["out"][:4], rtol=2e-4, atol=2e-5)


def test_spatial_attention_kernel_vs_fp64():
    """stmp_spatial_attention_fwd alone: softmax_dim1(Vs @ sigmoid(LHS @ RHS + bs)) for 307 / 200 / 64 nodes against float64."""
    from pytorch_geometric_temporal_b200 import ops
    for n, B, T in ((307, 5, 12), (200, 3, 7), (64, 2, 12)):
        g = torch.Generator().manual_seed(n)
        lhs, rhs = torch.randn(B, n, T, generator=g) * 0.5, torch.randn(B, T, n, generator=g) * 0.5
        bs, Vs = torch.randn(n, n, generator=g) * 0.3, torch.randn(n, n, generator=g) * (1.5 / n ** 0.5)
        S = torch.softmax(Vs.double() @ torch.sigmoid(lhs.double() @ rhs.double() + bs.double()), dim=1)
        S32 = torch.softmax(Vs @ torch.sigmoid(lhs @ rhs + bs), dim=1)
        ST = ops.spatial_attention(lhs.to(DEV), rhs.to(DEV), bs.t().contiguous().to(DEV), ops.spatial_attention_prepack(Vs.to(DEV)))
        got = ST[:, :, :n].transpose(1, 2).cpu()
        err, err32 = (got.double() - S).abs().max().item(), (S32.double() - S).abs().max().item()
        assert err < 4 * err32 + 1e-7, (n, err, err32)
        assert torch.all(ST[:, :, n:] == 0)


def test_astgcn_factors_kernel_vs_torch_fp64():
    """stmp_astgcn_factors_fwd: temporal attention + X~ + spatial factors for F = 64 (vector path) and F = 1 (first block)."""
    from pytorch_geometric_temporal_b200 import ops
    for (B, N, T, Fi) in ((3, 307, 12, 64), (2, 307, 12, 1), (2, 50, 7, 8)):
        g = torch.Generator().manual_seed(N + Fi)
        r = lambda *s: torch.randn(*s, generator=g)
        X = r(B, N, T, Fi) * 0.7
        U1, U2, U3, be, Ve = r(N) * 0.1, r(Fi, N) * 0.2, r(Fi) * 0.5, r(1, T, T) * 0.3, r(T, T) * 0.5
        W1, W2, W3 = r(T) * 0.4, r(Fi, T) * 0.3, r(Fi) * 0.5
        d = lambda t: t.double()
        Xr = d(X).permute(0, 1, 3, 2)                                        # reference layout (B,N,F,T)
        lhs = torch.matmul(torch.matmul(Xr.permute(0, 3, 2, 1), d(U1)), d(U2))
        rhs = torch.matmul(d(U3), Xr)
        E = torch.softmax(torch.matmul(d(Ve), torch.sigmoid(torch.matmul(lhs, rhs) + d(be))), dim=1)
        Xt = torch.matmul(Xr.reshape(B, -1, T), E).reshape(B, N, Fi, T)
        want_l = torch.matmul(torch.matmul(Xt, d(W1)), d(W2))
        want_r = torch.matmul(d(W3), Xt).transpose(-1, -2)
        gl, gr, gE = ops.astgcn_factors(*(t.to(DEV) for t in (X, U1, U2, U3, be, Ve, W1, W2, W3)), want_E=True)
        # yardstick: the same chain in torch fp32 (the reference's arithmetic) against float64
        Xf = X.permute(0, 1, 3, 2)
        lhs32 = torch.matmul(torch.matmul(Xf.permute(0, 3, 2, 1), U1), U2)
        E32 = torch.softmax(torch.matmul(Ve, torch.sigmoid(torch.matmul(lhs32, torch.matmul(U3, Xf)) + be)), dim=1)
        Xt32 = torch.matmul(Xf.reshape(B, -1, T), E32).reshape(B, N, Fi, T)
        l32, r32 = torch.matmul(torch.matmul(Xt32, W1), W2), torch.matmul(W3, Xt32).transpose(-1, -2)
        for got, want, ref32 in ((gl, want_l, l32), (gr, want_r, r32), (gE, E, E32)):
            err, err32 = (got.cpu().double() - want).abs().max().item(), (ref32.double() - want).abs().max().item()
            assert err < 4 * err32 + 2e-6, (err, err32)


def test_gemm_blocks_shift_ln_epilogues_vs_torch():
    """stmp_gemm_blocks_f32: row-shifted blocks inside sequences (a 1x3 convolution without im2col), ragged widths, the
    ReLU + LayerNorm epilogue and a 12-column output -- against torch fp32 / fp64."""
    from pytorch_geometric_temporal_b200 import ops
    g = torch.Generator().manual_seed(0)
    B, T, C = 37, 12, 64                                  # 444 rows: not a multiple of the 128-row tile
    Xh, X1 = torch.randn(B, T, C, generator=g), torch.randn(B, T, 1, generator=g)
    Wt, Wr = torch.randn(C, C, 3, generator=g) * 0.1, torch.randn(C, 1, generator=g)
    bias, gamma, beta = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    conv = torch.nn.functional.conv1d(Xh.transpose(1, 2), Wt, padding=1).transpose(1, 2) + X1 @ Wr.t() + bias
    want = torch.nn.functional.layer_norm(torch.relu(conv), (C,), gamma, beta, 1e-5)
    packed = ops.gemm_blocks_prepack([Wt[:, :, j].t().contiguous().to(DEV) for j in range(3)] + [Wr.t().contiguous().to(DEV)])
    xh, x1 = Xh.to(DEV).reshape(B * T, C), X1.to(DEV).reshape(B * T, 1)
    got = ops.gemm_blocks([(xh, C, -1), (xh, C, 0), (xh, C, 1), (x1, 1, 0)], packed, 64, 64, bias.to(DEV), ops.EPI_RELU_LN,
                          gamma.to(DEV), beta.to(DEV), 1e-5, seq=T)
    _close(got, want.reshape(B * T, C), rtol=1e-4, atol=2e-5)
    # plain / ReLU epilogues with a narrow output (final convolution: 12 columns of a 16-column product)
    W = torch.randn(3 * C, 16, generator=g) * 0.1
    packed = ops.gemm_blocks_prepack([W[C * i:C * i + C].to(DEV) for i in range(3)])
    rows = torch.randn(200, 3 * C, generator=g)
    rd = rows.to(DEV)
    b16 = torch.randn(16, generator=g)
    blocks = [(rd[:, C * i:C * i + C], C, 0) for i in range(3)]
    _close(ops.gemm_blocks(blocks, packed, 16, 12, b16.to(DEV), ops.EPI_BIAS), (rows @ W + b16)[:, :12], rtol=1e-4, atol=2e-5)
    _close(ops.gemm_blocks(blocks, packed, 16, 16, b16.to(DEV), ops.EPI_RELU), torch.relu(rows @ W + b16), rtol=1e-4, atol=2e-5)


def test_chebconv_attention_errors_and_repr():
    conv = ChebConvAttention(2, 3, 3, None).to(DEV)
    assert repr(conv) == "ChebConvAttention(2, 3, K=3, normalization=None)"   # test/attention_test.py:197
    x, S = torch.randn(2, 4, 2, device=DEV), torch.rand(2, 4, 4, device=DEV)
    ei = torch.tensor([[0, 0, 0, 1, 2, 3], [1, 2, 3, 0, 0, 0]], device=DEV)
    with pytest.raises(ValueError):
        conv(x, ei, S)                       # lambda_max mandatory unless "sym" (astgcn.py:135-139)
    assert conv(x, ei, S, lambda_max=2.0).shape == (2, 4, 3)
    with pytest.raises(AssertionError):
        ChebConvAttention(2, 3, 3, "bogus")


@pytest.mark.parametrize("norm", ["sym", None, "rw"])
def test_chebconv_attention_per_graph_lambda_max_vs_oracle(norm):
    """Multi-graph mini-batch: node->graph `batch` vector + one lambda_max per graph (test/attention_test.py:205-218;
    astgcn.py:98-99) -> stmp_plan_create_pergraph."""
    from oracle import attention as A
    torch.manual_seed(0)
    conv = ChebConvAttention(5, 7, K=3, normalization=norm)
    batch = torch.tensor([0, 0, 0, 1, 1, 1, 1])
    ei = torch.tensor([[0, 1, 1, 2, 3, 4, 5, 6, 3, 6], [1, 0, 2, 1, 4, 3, 6, 5, 6, 3]])
    ew = torch.rand(ei.size(1)) + 0.1
    x, S = torch.randn(3, 7, 5), torch.softmax(torch.rand(3, 7, 7), dim=1)
    lam = torch.tensor([2.0, 3.0])
    with torch.no_grad():
        want = A.cheb_conv_attention(conv.state_dict(), x, ei, S, norm, ew, lam, batch)
        want4 = A.cheb_conv_attention(conv.state_dict(), x, ei, S, norm, ew, torch.tensor(2.0), batch) if norm == "sym" else None
        m = conv.to(DEV)
        got = m(x.to(DEV), ei.to(DEV), S.to(DEV), ew.to(DEV), batch.to(DEV), lam.to(DEV))
        _close(got, want)
        if norm == "sym":                      # `batch` without lambda_max: the default 2.0 for every graph (out4 of the reference test)
            _close(m(x.to(DEV), ei.to(DEV), S.to(DEV), ew.to(DEV), batch.to(DEV)), want4)


def test_chebconv_layer_per_graph_lambda_max_vs_oracle():
    """PyG ChebConv with `batch` + lambda_max vector (`lambda_max[batch[edge_index[0]]]`)."""
    from oracle import pyg
    from pytorch_geometric_temporal_b200.nn.recurrent._cheb import ChebConv
    torch.manual_seed(0)
    batch = torch.tensor([0, 0, 0, 1, 1, 1, 1])
    ei = torch.tensor([[0, 1, 1, 2, 3, 4, 5, 6, 3, 6], [1, 0, 2, 1, 4, 3, 6, 5, 6, 3]])
    ew = torch.rand(ei.size(1)) + 0.1
    x = torch.randn(7, 5)
    lam = torch.tensor([2.0, 3.5])
    for norm in ("sym", "rw", None):
        conv = ChebConv(5, 6, 3, normalization=norm)
        ref = pyg.ChebConv(5, 6, 3, normalization=norm)
        ref.load_state_dict(conv.state_dict())
        with torch.no_grad():
            want = ref(x, ei, ew, batch, lam)
            got = conv.to(DEV)(x.to(DEV), ei.to(DEV), ew.to(DEV), batch.to(DEV), lam.to(DEV))
        _close(got, want)


def test_astgcn_backward_runs_and_matches_oracle_grad(golden_dir):
    """Training path: gradients flow through the attention-weighted SpMM (stmp_spmm_att_grad)."""
    from oracle import attention as A
    g = _load(golden_dir, "astgcn_small")
    c = g["cases"]["sym"]
    p = {k: v.clone().requires_grad_(True) for k, v in c["state"].items()}
    out = A.astgcn(p, c["X"], g["edge_index"], g["ctor"]["nb_block"], "sym", g["ctor"]["time_strides"])
    out.square().sum().backward()
    m = ASTGCN(**g["ctor"], normalization="sym").to(DEV)
    m.load_state_dict(c["state"])
    m(c["X"].to(DEV), g["edge_index"].to(DEV)).square().sum().backward()
    for k, prm in m.named_parameters():
        _close(prm.grad, p[k].grad, rtol=2e-3, atol=2e-4)


# ---- the generic fused graph-GRU kernel (stmp_gru_seq_fwd, wgmma) behind GConvGRU / TGCN / A3TGCN -----------------
def _metr():
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    return torch.from_numpy(ei), torch.from_numpy(ew)


@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("norm", ["sym", "rw"])
def test_gconv_gru_fused_tc_vs_oracle(K, norm):
    ei, ew = _metr()
    torch.manual_seed(K)
    m = GConvGRU(4, 32, K, normalization=norm)
    for p in m.parameters():   # non-zero biases
        if p.dim() == 1:
            torch.nn.init.uniform_(p, -0.5, 0.5)
    X, H = torch.randn(207, 4), torch.randn(207, 32) * 0.5
    lm = None if norm == "sym" else torch.tensor(2.4)
    want = R.gconv_gru_cell(m.state_dict(), X, ei, ew, H, lm, norm)
    mg = m.to(DEV)
    args = (X.to(DEV), ei.to(DEV), ew.to(DEV), H.to(DEV), None if lm is None else lm.to(DEV))
    with torch.no_grad():
        got = mg(*args)                       # builds the plan, packs the weights
        n0 = _lib.launch_count()
        got2 = mg(*args)                      # plan + pack cached
        assert _lib.launch_count() - n0 == 1  # ONE fused launch for the whole cell
    _close(got, want); _close(got2, want)
    _close(mg(*args), want)                   # tiled / autograd path


@pytest.mark.parametrize("improved", [False, True])
def test_tgcn_family_fused_tc_vs_oracle(improved):
    ei, ew = _metr()
    torch.manual_seed(3)
    m = TGCN(2, 32, improved=improved)
    for p in m.parameters():
        if p.dim() == 1:
            torch.nn.init.uniform_(p, -0.5, 0.5)
    X, H = torch.randn(207, 2), torch.randn(207, 32) * 0.5
    want = R.tgcn_cell(m.state_dict(), X, ei, ew, H, improved)
    with torch.no_grad():
        _close(m.to(DEV)(X.to(DEV), ei.to(DEV), ew.to(DEV), H.to(DEV)), want)
        _close(m(X.to(DEV), ei.to(DEV), ew.to(DEV)), R.tgcn_cell(m.cpu().state_dict(), X, ei, ew, None, improved))
    m2 = TGCN2(2, 32, 5, improved=improved)
    Xb, Hb = torch.randn(5, 207, 2), torch.randn(5, 207, 32) * 0.5
    want2 = R.tgcn_cell(m2.state_dict(), Xb, ei, ew, Hb, improved)
    with torch.no_grad():
        _close(m2.to(DEV)(Xb.to(DEV), ei.to(DEV), ew.to(DEV), Hb.to(DEV)), want2)


def test_a3tgcn_fused_tc_vs_oracle():
    ei, ew = _metr()
    torch.manual_seed(5)
    m = A3TGCN2(2, 32, 12, 4)
    X, H = torch.randn(4, 207, 2, 12), torch.randn(4, 207, 32) * 0.3
    want, wantH = R.a3tgcn(m.state_dict(), X, ei, ew), R.a3tgcn(m.state_dict(), X, ei, ew, H)
    mg = m.to(DEV)
    a = (X.to(DEV), ei.to(DEV), ew.to(DEV))
    with torch.no_grad():
        got = mg(*a)
        n0 = _lib.launch_count()
        gotH = mg(*a, H.to(DEV))
        assert _lib.launch_count() - n0 == 1   # 12 periods x 4 rows = 48 one-step windows in ONE launch
    _close(got, want); _close(gotH, wantH)
    m1 = A3TGCN(2, 32, 6)
    X1, H1 = torch.randn(207, 2, 6), torch.randn(207, 32) * 0.3
    want1 = R.a3tgcn(m1.state_dict(), X1, ei, ew, H1)
    with torch.no_grad():
        _close(m1.to(DEV)(X1.to(DEV), ei.to(DEV), ew.to(DEV), H1.to(DEV)), want1)


def test_masked_mae_fused_matches_reference_form():
    """stmp_masked_mae_fwd/bwd vs the op-for-op loss of examples/indexBatching/DCRNN/utils.py:10-18 (value and gradient),
    incl. masked zeros, NaN predictions, an all-zero target (0/0 mask -> loss 0) and a non-contiguous prediction."""
    from pytorch_geometric_temporal_b200 import distributed as D
    torch.manual_seed(0)
    for shape, frac_zero, nan in (((64, 207), 0.2, False), ((7, 13), 0.5, True), ((300001,), 0.0, False), ((5, 9), 1.0, False)):
        y = torch.randn(shape, device=DEV)
        y[torch.rand(shape, device=DEV) < frac_zero] = 0.0
        p = torch.randn(shape, device=DEV)
        if nan:
            p.view(-1)[3] = float("nan")
        pa, pb = p.clone().requires_grad_(True), p.clone().requires_grad_(True)
        la, lb = D.masked_mae_loss(pa, y), D.masked_mae_loss_reference(pb, y)
        assert torch.allclose(la, lb, rtol=1e-5, atol=1e-7), (float(la), float(lb))
        (la * 3.0).backward(); (lb * 3.0).backward()
        ga, gb = pa.grad, torch.nan_to_num(pb.grad, nan=0.0)      # the reference's where() leaves NaN grads at NaN terms
        assert torch.allclose(torch.nan_to_num(ga, nan=0.0), gb, rtol=1e-5, atol=1e-9)
    base = torch.randn(64, 207, 2, device=DEV)
    pa = base.clone().requires_grad_(True)
    y = torch.randn(64, 207, device=DEV)
    la = D.masked_mae_loss(pa[..., 0], y)                        # strided view
    lb = D.masked_mae_loss_reference(base[..., 0], y)
    assert torch.allclose(la, lb, rtol=1e-5)
    la.backward()
    assert pa.grad[..., 1].abs().max() == 0 and pa.grad[..., 0].abs().max() > 0


@pytest.mark.parametrize("fused", [True, False])
def test_a3tgcn2_config3_training_gradients_vs_reference_golden(golden_dir, fused):
    """Training call of the reference's A3TGCN2 example (no incoming state) at the PEMS-BAY shape: output and the gradient of EVERY
    parameter against the unmodified reference's autograd (tests/golden/make_goldens_r2.py::a3tgcn2_cfg3_grads) -- through the fused
    forward + hand-written backward (stmp_tgcn_attn_fwd / _bwd) and through the op-for-op autograd path; same for a TGCN2 cell."""
    from pytorch_geometric_temporal_b200.nn.recurrent import TGCN2
    g = _load(golden_dir, "a3tgcn2_cfg3_grads")
    ei, ew, X = (g[k].to(DEV) for k in ("edge_index", "edge_weight", "X"))
    m = A3TGCN2(2, 32, 12, 8).to(DEV)
    m.load_state_dict(g["state"])
    m._base_tgcn.fused_training = fused
    c0 = _lib.path_counters()
    out = m(X, ei, ew)
    w = torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)
    (out * w).sum().backward()
    assert (_ran(c0, "k_tgcn_attn_bwd") == 1) == fused
    _close(out, g["out"])
    for k, p in m.named_parameters():
        ref = g["grads"][k]
        assert p.grad is not None, k
        _close(p.grad, ref, 1e-3, 1e-3 * ref.abs().max().item() + 1e-6)
    c2 = TGCN2(2, 32, 8).to(DEV)
    c2.load_state_dict(g["state_cell"])
    c2.fused_training = fused
    c0 = _lib.path_counters()
    cell = c2(X[..., 3], ei, ew)
    (cell * w).sum().backward()
    assert (_ran(c0, "k_tgcn_attn_bwd") == 1) == fused
    _close(cell, g["cell"])
    for k, p in c2.named_parameters():
        ref = g["grads_cell"][k]
        _close(p.grad, ref, 1e-3, 1e-3 * ref.abs().max().item() + 1e-6)


def test_a3tgcn2_training_step_with_state_or_input_grad_takes_the_autograd_path():
    """An incoming state or a gradient w.r.t. X is outside the hand-written backward: those calls stay on the differentiable op-for-op path."""
    ei, ew, _ = synthetic.pems_bay_like(0, 16)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    torch.manual_seed(0)
    m = A3TGCN2(2, 32, 12, 4).to(DEV)
    X = torch.randn(4, 325, 2, 12, device=DEV)
    H = torch.randn(4, 325, 32, device=DEV) * 0.5
    c0 = _lib.path_counters()
    m(X, ei, ew, H).sum().backward()
    Xg = X.clone().requires_grad_(True)
    m(Xg, ei, ew).sum().backward()
    assert Xg.grad is not None and _ran(c0, "k_tgcn_attn_bwd") == 0
