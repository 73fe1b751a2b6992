"""One small invocation of every hand-synchronised kernel (mbarriers, wgmma, proxy fences, TMA bulk copies, cluster pairs)
for compute-sanitizer:   tools/sanitize.sh   runs this under --tool memcheck and --tool racecheck."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pytorch_geometric_temporal_b200 import _lib, ops                                        # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic                               # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN                              # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN2, BatchedDCRNN, DyGrEncoder, EvolveGCNH, EvolveGCNO, GCLSTM, GConvGRU, GConvLSTM, LRGCN, MPNNLSTM, TGCN2   # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import AGCRN                                # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import GMAN, MTGNN                          # noqa: E402
from pytorch_geometric_temporal_b200.nn.hetero import HeteroGCLSTM                          # noqa: E402

dev = torch.device("cuda")
torch.manual_seed(0)
ei, ew, series = synthetic.metr_la_like(0, 40)
ei_t, ew_t = torch.from_numpy(ei).to(dev), torch.from_numpy(ew).to(dev)
X = torch.from_numpy(series[:36]).reshape(3, 12, 207, 2).to(dev)
m = BatchedDCRNN(2, 32, 2).to(dev)
with torch.no_grad():
    m(X, ei_t, ew_t)                                             # k_dcrnn_seq_tc (wgmma, TMA images, MMA groups)
m(X[:2], ei_t, ew_t).square().mean().backward()                  # + stash; CTA-pair (cluster) forward and backward, k_dcrnn_bwd_basis, k_dcrnn_wgrad_tc
for opt in ("dcrnn_fwd_split", "dcrnn_bwd_split", "dcrnn_wgrad_tc"):
    _lib.set_option(opt, 0)
with torch.no_grad():
    m(X, ei_t, ew_t)                                             # one CTA per window
m(X[:2], ei_t, ew_t).square().mean().backward()                  # one-CTA backward, FFMA weight-gradient kernel
for opt in ("dcrnn_fwd_split", "dcrnn_bwd_split", "dcrnn_wgrad_tc"):
    _lib.set_option(opt, 1)
from pytorch_geometric_temporal_b200 import distributed as D   # noqa: E402
sync = D.FlatGradSync(m.parameters())
opt_ = D.FlatAdam(sync, lr=1e-3)
m(X[:2], ei_t, ew_t).square().mean().backward()
opt_.step()                                                      # k_adam_flat
with torch.no_grad():
    BatchedDCRNN(2, 16, 3).to(dev)(X[:2], ei_t, ew_t)            # k_dcrnn_seq (FFMA2, TMA window buffers)
    g = GConvGRU(2, 32, 2).to(dev)
    g(X[0, 0], ei_t, ew_t)                                       # generic graph-GRU entry (one operator)
    e3, w3, _ = synthetic.pems_bay_like(0, 16)
    a3 = A3TGCN2(2, 32, 12, 4).to(dev)
    a3(torch.randn(4, 325, 2, 12, device=dev), torch.from_numpy(e3).to(dev), torch.from_numpy(w3).to(dev),
       torch.randn(4, 325, 32, device=dev))                      # k_tgcn_attn (TMA-staged X)
with torch.enable_grad():
    a3(torch.randn(4, 325, 2, 12, device=dev), torch.from_numpy(e3).to(dev), torch.from_numpy(w3).to(dev)).square().mean().backward()   # k_tgcn_attn_bwd
    t2, h = TGCN2(4, 32, 3).to(dev), None
    for t in range(3):                                           # TGCN2 training with the state carried: step 0 k_tgcn_attn_bwd,
        h = t2(torch.randn(3, 207, 4, device=dev), ei_t, ew_t, h)   # then k_tgcn_cell_bwd (TMA-staged X, staged Bm) + its reduce
    h.square().mean().backward()
    for n in (207, 40000):                                       # 64 channels: k_tgcn_wide_attn (Bm staged next to X), k_tgcn_attn_bwd<NQ, 2>,
        en = torch.randint(0, n, (2, 4 * n), device=dev)         # k_tgcn_wide_cell_bwd + the 64-wide weight-gradient kernels; X staged at
        a64, t64, h = A3TGCN2(2, 64, 12, 2).to(dev), TGCN2(4, 64, 2).to(dev), None   # 207 nodes, gathered from global memory at 40 000
        a64(torch.randn(2, n, 2, 12, device=dev), en).square().mean().backward()
        with torch.no_grad():
            a64(torch.randn(2, n, 2, 12, device=dev), en, None, torch.randn(2, n, 64, device=dev))
        for t in range(2):
            h = t64(torch.randn(2, n, 4, device=dev), en, None, h)
        h.square().mean().backward()
    for K in (1, 2):                                           # GConvGRU training: stashing forward, k_gru_pack_bwd_weights,
        gg = GConvGRU(2, 32, K).to(dev)                          # k_gru_bwd_basis, k_gru_bwd_seq (CTA pair), k_dcrnn_wgrad_tc, k_gru_wgrad_reduce
        gg(X[0, 0], ei_t, ew_t, torch.randn(207, 32, device=dev, requires_grad=True)).square().mean().backward()
    # the generic graph-GRU envelope (tests/test_gpu_gru_seq_envelope.py): K = 1 (n_ops = 0) with H = None and dX; the one-CTA backward
    # at one operator, SMs / 2 + 1 windows; a forward from one h0 shared by every window
    GConvGRU(2, 32, 1).to(dev)(X[0, 0].clone().requires_grad_(True), ei_t, ew_t).square().mean().backward()
    nb = torch.cuda.get_device_properties(dev).multi_processor_count // 2 + 1
    pg, (wg_, bg, ig), (sg, prm) = gg._cheb_plan(ei_t, ew_t, 207, "sym", None), gg._packed(), gg._param_spec()
    xb = torch.randn(nb, 2, 207, 2, device=dev, requires_grad=True)
    ops.gru_seq_train(pg, 1, xb, torch.randn(nb, 207, 32, device=dev, requires_grad=True), wg_, bg, ig, sg, prm).square().mean().backward()
    with torch.no_grad():
        ops.gru_seq_fwd(pg, 1, xb.detach(), wg_, bg, h0=torch.randn(207, 32, device=dev), h0_shared=True, wimage=ig)
    ring = torch.arange(301, device=dev)
    e_ring = torch.cat([torch.stack([ring, (ring + 1) % 301]), torch.stack([(ring + 5) % 301, ring])], dim=1)
    gr = GConvGRU(14, 32, 2).to(dev)                             # 301 nodes: the row-split cell kernels (k_gru_rows_*), H given and None,
    xr = torch.randn(301, 14, device=dev, requires_grad=True)    # X gradient: k_dcrnn_wgrad + k_gru_rows_wgrad_reduce
    gr(xr, e_ring, None, torch.randn(301, 32, device=dev, requires_grad=True)).square().mean().backward()
    gr(xr, e_ring, None).square().mean().backward()
    with torch.no_grad():
        gr(xr, e_ring, None, torch.randn(301, 32, device=dev))
    for cls in (GConvLSTM, GCLSTM):                              # the row-split LSTM cell (k_lstm_rows_*), both bases: n_ops 0 and 1,
        for K in (1, 2):                                         # H / C given and None, k_dcrnn_wgrad<64> + k_lstm_rows_wgrad_reduce
            gl = cls(14, 32, K).to(dev)
            hc = [torch.randn(301, 32, device=dev, requires_grad=True) for _ in range(2)]
            sum(t.square().mean() for t in gl(xr, e_ring, None, *hc)).backward()
            sum(t.square().mean() for t in gl(xr, e_ring, None)).backward()
            with torch.no_grad():
                gl(xr, e_ring, None, hc[0].detach(), hc[1].detach())
    t_ring = torch.arange(e_ring.size(1), device=dev) % 3             # relation 0, 1 and a type that matches neither
    for co, R in ((32, 2), (64, 1)):                             # LRGCN: the relational plan (k_flag_relation, k_mean_vals) and the two-
        lr = LRGCN(14, co, R, 2).to(dev)                         # operator cell (k_lstm_rows_*<.., 2>, k_wide_rows_wgrad<2> + reduce)
        hc = [torch.randn(301, co, device=dev, requires_grad=True) for _ in range(2)]
        sum(t.square().mean() for t in lr(xr, e_ring, t_ring, *hc)).backward()
        sum(t.square().mean() for t in lr(xr, e_ring, t_ring)).backward()
    w_ring = torch.rand(e_ring.size(1), device=dev)
    for aggr, C, Lg in (("mean", 16, 2), ("max", 32, 3)):          # DyGrEncoder: the gated plan (k_gated_vals), k_ggc_rows_msg /
        dy = DyGrEncoder(C, Lg, aggr, 32, 1).to(dev)            # _fwd / _bwd (with dX) / _wgrad + reduce, and the LSTM cell with n_ops = 0
        xg = xr[:, :C].detach().clone().requires_grad_(True)    # (C = 16) or the cuDNN LSTM (C = 32)
        sum(t.square().mean() for t in dy(xg, e_ring, w_ring)).backward()
    for eg in (EvolveGCNO(14).to(dev), EvolveGCNH(301, 14).to(dev)):    # EvolveGCN: k_egcn_fwd / k_egcn_score + k_egcn_fwd_topk,
        xe = xr.detach().clone().requires_grad_(True)                 # k_egcn_bwd_rows (with dX) and k_egcn_wgrad(_topk), two calls chained
        (eg(xe, e_ring, w_ring).square().mean() + eg(xe, e_ring, w_ring).mean()).backward()
        with torch.no_grad():
            eg(xr, e_ring, None)
    mp = MPNNLSTM(14, 32, 301, 1, 0.5).to(dev)                  # MPNN-LSTM: k_mpnn_conv1 / _conv2 / _lstm in training mode (dropout
    with torch.no_grad():                                        # bits, running statistics) and eval mode, and the backward with dX
        mp(xr, e_ring, w_ring)
        mp.eval()(xr, e_ring, None)
    mp.train()(xr, e_ring, w_ring).square().mean().backward()
    for K in (1, 3):                                             # AGCRN: every k_agcrn_* kernel, partial tiles (N = 67, B = 3), with and
        ag = AGCRN(67, 5, 7, K, 6).to(dev)                       # without H, the backward with every gradient
        xa, ea = torch.randn(3, 67, 5, device=dev), torch.randn(67, 6, device=dev, requires_grad=True)
        ha = ag(xa.requires_grad_(True), ea)
        ag(xa, ea, ha).square().mean().backward()
        with torch.no_grad():
            ag(xa, ea)
    for K, d, N, mask in ((8, 8, 131, True), (13, 2, 5, False)):  # GMAN: every k_gman_attn_* kernel at widths 8 and 16 (13 padded), a
        gm = GMAN(1, K, d, 5, 0.1, 12, True, mask).to(dev)        # partial query / key tile (N = 131), the masked short kernels and
        xg, se = torch.rand(2, 5, N, device=dev), torch.randn(N, K * d, device=dev)   # their backwards
        te = torch.randint(0, 12, (2, 9, 2), device=dev).float()
        gm(xg, se, te).square().mean().backward()
        with torch.no_grad():
            gm.eval()(xg, se, te)
    for n, k, depth, T in ((37, 5, 2, 13), (70, 64, 1, 40)):    # MTGNN: every k_mtgnn_* kernel; a partial bitmap word column (37, 70
        mt = MTGNN(True, True, depth, n, [2, 3], 3, 0.0, k, 6, 1, 4, 5, 6, 8, T, 2, 3, 2, 0.05, 3.0, True).to(dev)   # nodes), T below
        xm = torch.rand(2, 2, n, T, device=dev)                  # and above a warp, the graph backward; then a predefined A
        mt(xm).square().mean().backward()
        with torch.no_grad():
            MTGNN(True, False, depth, n, [2, 3], 3, 0.0, k, 6, 1, 4, 5, 6, 8, T, 2, 3, 2, 0.05, 3.0, True).to(dev)(
                xm, (torch.rand(n, n, device=dev) < 0.2).float())
    for out, rel in ((32, 4), (64, 1)):                          # HeteroGCLSTM: k_hetero_lstm_fwd at both widths, H None and carried,
        ht = {"a": (301, 5), "b": (17, 32)}                      # partial tiles and a type change inside a CTA's tiles
        eh = {("a", "r", "b"): torch.stack([torch.arange(60) % 301, torch.arange(60) % 17]).to(dev),
              ("b", "r", "a"): torch.stack([torch.arange(400) % 17, torch.arange(400) % 301]).to(dev)}
        for k in range(1, rel):
            eh[("b", f"s{k}", "b")] = torch.stack([torch.arange(30) % 17, (torch.arange(30) * 7) % 17]).to(dev)
        hg = HeteroGCLSTM({t: c for t, (_, c) in ht.items()}, out, (list(ht), list(eh))).to(dev)
        xh = {t: torch.randn(n, c, device=dev) for t, (n, c) in ht.items()}
        with torch.no_grad():
            hg(xh, eh, *hg(xh, eh))
    for cin, T in ((2, 3), (4, 1)):                              # 301 nodes: the row-split DCRNN (k_dcrnn_rows_*), T = 1 and T > 1, with and
        dr = BatchedDCRNN(cin, 32, 2).to(dev)                    # without dX (k_dcrnn_rows_bwd_x), k_dcrnn_wgrad_tc + k_dcrnn_wgrad_reduce
        xd = torch.randn(2, T, 301, cin, device=dev)
        dr(xd.clone().requires_grad_(True), e_ring, None).square().mean().backward()
        dr(xd, e_ring, None).square().mean().backward()
        with torch.no_grad():
            dr(xd, e_ring, None)
    e_big = torch.stack([torch.arange(1100), (torch.arange(1100) + 1) % 1100]).to(dev)     # 1100 nodes: above the one-SM narrow kernels
    for cin, cout, K, T in ((2, 2, 3, 3), (1, 3, 2, 1), (2, 1, 1, 2)):   # the narrow row-split DCRNN (k_dcrnn_nrows_*), with and without dX
        dn = BatchedDCRNN(cin, cout, K).to(dev)
        xn = torch.randn(3, T, 1100, cin, device=dev)
        dn(xn.clone().requires_grad_(True), e_big, None).square().mean().backward()
        dn(xn, e_big, None).square().mean().backward()
        with torch.no_grad():
            dn(xn, e_big, None)
    for cin, K, T in ((2, 3, 3), (3, 2, 1)):                     # 301 nodes, 3 windows (a partial last warp): the 64-wide row-split DCRNN
        dw = BatchedDCRNN(cin, 64, K).to(dev)                    # (k_dcrnn_wrows_*), T = 1 and T > 1, with and without dX
        xw = torch.randn(3, T, 301, cin, device=dev)
        dw(xw.clone().requires_grad_(True), e_ring, None).square().mean().backward()
        dw(xw, e_ring, None).square().mean().backward()
        with torch.no_grad():
            dw(xw, e_ring, None)
with torch.no_grad():
    e4 =torch.from_numpy(synthetic.pems04_like(0)).to(dev)
    ASTGCN(2, 1, 3, 64, 64, 1, 12, 12, 307, normalization="sym").to(dev)(torch.randn(2, 307, 1, 12, device=dev), e4)   # k_gemm_blocks x7
    e7 = torch.from_numpy(synthetic.pems07_like(0)).to(dev)
    ASTGCN(1, 1, 3, 64, 64, 1, 12, 12, 883, normalization="sym").to(dev)(torch.randn(2, 883, 1, 12, device=dev), e7)   # k_spatt_tiles x4 columns + k_spatt_norm
    ops.spatial_attention_tiled(torch.randn(1, 70, 5, device=dev), torch.randn(1, 5, 70, device=dev), torch.randn(70, 70, device=dev),
                                ops.spatial_attention_prepack(torch.randn(70, 70, device=dev)))   # one column tile, partial row tile, T < 12
    # the ASTGCN envelope (tests/test_gpu_astgcn_envelope.py): a scalar factors instance (F = 2), the 8-chunk one-tile attention
    # (100 nodes, T = 7), and a forward at in_channels 3 (torch factors), K = 1, T = 1 with 129 outputs (the 20-chunk EPI_BIAS instance)
    ops.astgcn_factors(torch.randn(2, 40, 7, 2, device=dev), *[torch.randn(*s, device=dev) for s in ((40,), (2, 40), (2,), (7, 7), (7, 7),
                                                                                                      (7,), (2, 7), (2,))])
    ops.spatial_attention(torch.randn(2, 100, 7, device=dev), torch.randn(2, 7, 100, device=dev), torch.randn(100, 100, device=dev),
                          ops.spatial_attention_prepack(torch.randn(100, 100, device=dev)))
    r50 = torch.arange(50, device=dev)
    ASTGCN(1, 3, 1, 64, 64, 1, 129, 1, 50, normalization="sym").to(dev)(torch.randn(2, 50, 3, 1, device=dev),
                                                                         torch.stack([r50, (r50 + 1) % 50]))
    eg, wg = synthetic.large_graph(2000, 20000, 0)
    eg, wg = torch.from_numpy(eg).to(dev), torch.from_numpy(wg).to(dev)
    lstm = GConvLSTM(64, 64, 3).to(dev)
    lstm(torch.randn(2000, 64, device=dev), eg, wg)              # k_spmm + k_gemm_split<LSTM epilogue>
    nm = BatchedDCRNN(2, 2, 3).to(dev)
    _lib.set_option("dcrnn_narrow_pack", 3)
    nm(X[:5, :4], ei_t, ew_t)                                    # k_dcrnn_narrow_seq, 3 windows per CTA (one group half empty)
    _lib.set_option("dcrnn_narrow_pack", 0)
(nm(X[:3, :4], ei_t, ew_t) * torch.randn(3, 4, X.size(2), 2, device=dev)).sum().backward()   # k_dcrnn_narrow_bwd, one window per CTA
_lib.set_option("dcrnn_narrow_pack", 2)
(nm(X[:3, :4], ei_t, ew_t) * torch.randn(3, 4, X.size(2), 2, device=dev)).sum().backward()   # packed: 2 windows per CTA, 2 tasks per thread
e8 = torch.stack([torch.arange(40), (torch.arange(40) * 7 + 1) % 40]).to(dev)
nm8 = BatchedDCRNN(4, 4, 3).to(dev)
_lib.set_option("dcrnn_narrow_pack", 8)
(nm8(torch.randn(10, 3, 40, 4, device=dev), e8, torch.ones(40, device=dev)) ** 2).sum().backward()   # CP = 8, 8 windows per CTA, tail group, 320 tasks: the backward at 2 per thread
_lib.set_option("dcrnn_narrow_pack", 0)
with torch.no_grad():
    r600 = torch.arange(600, device=dev)
    nm8(torch.randn(2, 3, 600, 4, device=dev), torch.stack([r600, (r600 * 7 + 1) % 600]), torch.ones(600, device=dev))   # CP = 8, 4 tasks per thread
x = torch.randn(2, 2000, 64, device=dev, requires_grad=True)
h, c = lstm(x, eg, wg)
(h.sum() + c.sum()).backward()                                   # _LstmCellFn backward: k_gemm_split, k_lstm_gate_bwd, transposed SpMM
# a state of (N, out) shared by a batch of 2 windows (tests/test_gpu_cheb_lstm_envelope.py): the fused GEMM + gate epilogue, the
# pointwise gates and _LstmCellFn at K = 4, whose adjoint loop runs twice, each with dH / dC summed over the windows
hs = torch.randn(2000, 32, device=dev, requires_grad=True)
cs = torch.randn(2000, 32, device=dev, requires_grad=True)
with torch.no_grad():
    lstm(torch.randn(2, 2000, 64, device=dev), eg, wg, torch.randn(2000, 64, device=dev), torch.randn(2000, 64, device=dev))
    GCLSTM(3, 33, 2).to(dev)(torch.randn(2, 2000, 3, device=dev), eg, wg, torch.randn(2000, 33, device=dev), torch.randn(2000, 33, device=dev))
sum(t.sum() for t in GConvLSTM(32, 32, 4).to(dev)(torch.randn(2, 2000, 32, device=dev, requires_grad=True), eg, wg, hs, cs)).backward()
# adversarial geometries (tests/test_gpu_graph_geometry.py): a 128-edge row in the second row tile, a backward that reads the global CSR,
# the FFMA kernel's 7-rows-per-thread mapping
r129 = torch.arange(129, device=dev)
e_hub = torch.cat([torch.stack([r129, (r129 + 1) % 129]), torch.stack([r129[:-1], torch.full((128,), 128, device=dev)])], dim=1)
mh = BatchedDCRNN(3, 32, 2).to(dev)
mh(torch.randn(2, 4, 129, 3, device=dev), e_hub, torch.ones(e_hub.size(1), device=dev)).square().mean().backward()   # cluster pairs
r207 = torch.arange(207, device=dev)
pairs = torch.randperm(207 * 207, generator=torch.Generator().manual_seed(0))[:2107].to(dev)
e_dense = torch.cat([torch.stack([r207, (r207 + 1) % 207]), torch.stack([pairs // 207, pairs % 207])], dim=1)
m(X[:2], e_dense, torch.ones(e_dense.size(1), device=dev)).square().mean().backward()   # k_dcrnn_bwd_seq[graph-global]
with torch.no_grad():
    r225 = torch.arange(225, device=dev)
    BatchedDCRNN(2, 32, 1).to(dev)(torch.randn(2, 12, 225, 2, device=dev), torch.stack([r225, (r225 + 1) % 225]),
                                   torch.ones(225, device=dev))  # k_dcrnn_seq, RT 7
# the row-split kernels below the modules' routing (tests/test_gpu_rows_envelope.py): 17 nodes, 3 windows -- 16-row tiles and 8-row
# warps that straddle windows, a partial last tile and warp, a partial lane group
from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnHoistedRowsFn, _DcrnnRowsFn   # noqa: E402
r17 = torch.arange(17, device=dev)
e17 = torch.cat([torch.stack([r17, (r17 + 1) % 17]), torch.stack([r17, (r17 + 5) % 17])], dim=1)
for cin, cout, K in ((3, 32, 2), (3, 64, 3), (2, 3, 3)):
    d17 = BatchedDCRNN(cin, cout, K).to(dev)
    p17 = d17._plan(e17, torch.ones(34, device=dev), 17)
    x17 = torch.randn(3, 3, 17, cin, device=dev, requires_grad=True)
    if cout == 32:
        _DcrnnRowsFn.apply(x17, *d17._params(), p17, d17._rows_packed()).square().mean().backward()
    else:
        _DcrnnHoistedRowsFn.apply(x17, *d17._params(), p17, K, d17._rows_packed()).square().mean().backward()
    with torch.no_grad():
        d17._rows_infer(p17, x17.detach())
g17 = GConvGRU(5, 32, 2).to(dev)
xg, hg = torch.randn(17, 5, device=dev, requires_grad=True), torch.randn(17, 32, device=dev, requires_grad=True)
ops.gru_rows_train(g17._cheb_plan(e17, None, 17, "sym", None), 1, xg, hg, *g17._rows_packed(), *g17._param_spec(rows=True)).square().mean().backward()
g64 = GConvGRU(5, 64, 2).to(dev)                                # the 64-wide cell at 17 nodes: partial last tile, every launch
xw, hw = torch.randn(17, 5, device=dev, requires_grad=True), torch.randn(17, 64, device=dev, requires_grad=True)
g64(xw, e17, None, hw).square().mean().backward()
with torch.no_grad():
    g64(xw, e17, None)
for cls in (GConvLSTM, GCLSTM):
    sum(t.square().mean() for t in cls(5, 32, 2).to(dev)(xg, e17, None, hg, torch.randn(17, 32, device=dev, requires_grad=True))).backward()
    l64 = cls(5, 64, 2).to(dev)                                 # the 64-wide LSTM cell at 17 nodes, H given and not
    sum(t.square().mean() for t in l64(xw, e17, None, hw, torch.randn(17, 64, device=dev, requires_grad=True))).backward()
    sum(t.square().mean() for t in l64(xw, e17, None)).backward()
    with torch.no_grad():
        l64(xw, e17, None, hw, hw)
# an ASTGCN training step (tests/test_gpu_attention_training.py): the attention hop forward, its transposed product and k_att_grad at
# the first block's F = 12 and the later blocks' F = 768; then ops.spmm on 2-D features and a transposed attention, F = 5 (VEC 1)
F.l1_loss(ASTGCN(2, 1, 3, 64, 64, 1, 12, 12, 307, normalization="rw").to(dev)(torch.randn(2, 307, 1, 12, device=dev), e4),
          torch.randn(2, 307, 12, device=dev)).backward()
p4 = ASTGCN(1, 1, 2, 64, 64, 1, 12, 12, 307)._blocklist[0]._chebconv_attention.to(dev)._plan(e4, None, 307, None)
s4 = torch.rand(1, 307, 307, device=dev).transpose(1, 2).requires_grad_(True)
ops.spmm(p4, 0, torch.randn(307, 5, device=dev, requires_grad=True), 0.5, att=s4).square().sum().backward()
torch.cuda.synchronize()
print("sanitize_smoke ok:", {k: v for k, v in _lib.path_counters().items() if k.startswith("k_") and v})
