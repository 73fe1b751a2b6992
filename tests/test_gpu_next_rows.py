"""GPU parity of the SURVEY 8f rank-1 modules (GCLSTM, STConv, MSTGCN) through the public modules -> C ABI, against
goldens generated from the unmodified reference (tests/golden/make_goldens_next.py).  Strict fp32: rtol 1e-4 / atol
1e-5 on outputs, 1e-3 / 1e-5 on gradients (same bars as the round-1 cells)."""
import os

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.attention import MSTGCN, STConv
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, ChebConv

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got = got.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _loss(outs):
    return sum((o * torch.linspace(-1, 1, o.numel(), device=o.device).view_as(o)).sum() for o in outs)


def _check_grads(m, want, rtol=1e-3, atol=1e-5):
    for k, p in m.named_parameters():
        _close(p.grad, want[k], rtol, atol)


def test_gc_lstm_goldens(golden_dir):
    g = _load(golden_dir, "gc_lstm_small")
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    for name, c in g["cases"].items():
        cin, cout = c.get("cin", 4), c.get("cout", 16)
        m = GCLSTM(cin, cout, c["K"], normalization=c["normalization"]).to(DEV)
        m.load_state_dict(c["state"])
        lm = None if c["lambda_max"] is None else c["lambda_max"].to(DEV)
        x, h, cc = c["X"].to(DEV), c["H"].to(DEV), c["C"].to(DEV)
        n0 = _lib.launch_count()
        with torch.no_grad():
            ho, co = m(x, ei, ew, h, cc, lm)                      # in-place basis + fused gate kernels / wgmma epilogue
            _close(ho, c["outH"]); _close(co, c["outC"])
            if "outH0" in c:
                ho, co = m(x, ei, lambda_max=lm)
                _close(ho, c["outH0"]); _close(co, c["outC0"])
        assert _lib.launch_count() > n0
        if "grads" in c:
            xg, hg, cg = (t.clone().requires_grad_(True) for t in (x, h, cc))
            ho, co = m(xg, ei, ew, hg, cg, lm)                    # autograd path
            _close(ho, c["outH"]); _close(co, c["outC"])
            _loss([ho, co]).backward()
            _check_grads(m, c["grads"])
            _close(xg.grad, c["gX"], 1e-3, 1e-5); _close(hg.grad, c["gH"], 1e-3, 1e-5); _close(cg.grad, c["gC"], 1e-3, 1e-5)


def test_gc_lstm_recurrence_matches_oracle_over_steps():
    """size-independent property: T chained cell calls stay on the oracle's trajectory (H, C fed back)."""
    ei, ew, series = synthetic.metr_la_like(seed=1, t_total=8)
    ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
    torch.manual_seed(0)
    m = GCLSTM(2, 32, 3)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    mg = m.to(DEV)
    eig, ewg = ei.to(DEV), ew.to(DEV)
    Hc = Cc = Hg = Cg = None
    for t in range(6):
        x = torch.from_numpy(series[t])
        Hc, Cc = R.gc_lstm_cell(sd, x, ei, ew, Hc, Cc)
        with torch.no_grad():
            Hg, Cg = mg(x.to(DEV), eig, ewg, Hg, Cg)
        _close(Hg, Hc); _close(Cg, Cc)


def test_stconv_goldens(golden_dir):
    g = _load(golden_dir, "stconv_small")
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    for name, c in g["cases"].items():
        m = STConv(K=c["K"], normalization=c["normalization"], **g["ctor"]).to(DEV)
        m.load_state_dict(c["state"])
        X = c["X"].to(DEV)
        m.eval()
        with torch.no_grad():
            _close(m(X, ei, ew), c["out_eval"])
            _close(m(X, ei), c["out_eval_noew"])
            n0 = _lib.launch_count()
            m(X, ei, ew)                                         # plan cached by now
        # (B, T') slices ride the batch axis: (K-1) SpMM launches per forward, not B*T'*(K-1)
        assert _lib.launch_count() - n0 == c["K"] - 1
        m.train()
        Xg = X.clone().requires_grad_(True)
        out = m(Xg, ei, ew)                                     # training-mode BatchNorm: batch statistics
        _close(out, c["out_train"])
        _loss([out]).backward()
        # training-mode BatchNorm backward is g - mean(g) - x^ mean(g x^): cancellation turns fp32 summation-order
        # differences (GPU vs CPU reductions) into absolute errors that scale with the LARGEST gradient entry, so the
        # bar is relative to the tensor's max: |err| <= 2e-4 * max|want|
        for k, p in m.named_parameters():
            _close(p.grad, c["grads"][k], 0.0, 2e-4 * float(c["grads"][k].abs().max()) + 1e-6)
        _close(Xg.grad, c["gX"], 0.0, 2e-4 * float(c["gX"].abs().max()) + 1e-6)


def test_stconv_batched_equals_per_slice_chebconv():
    """the folded (B*T') batch must equal the reference's per-slice loop bit for bit (same kernel, same row order)."""
    ei, ew, _ = synthetic.metr_la_like(seed=2, t_total=4)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    torch.manual_seed(0)
    conv = ChebConv(8, 8, 3).to(DEV)
    x = torch.randn(3, 5, 207, 8, device=DEV)
    with torch.no_grad():
        whole = conv(x.reshape(15, 207, 8), ei, ew).reshape(3, 5, 207, 8)
        for b in range(3):
            for t in range(5):
                assert torch.allclose(conv(x[b, t], ei, ew), whole[b, t], rtol=1e-6, atol=1e-6)


def test_mstgcn_goldens(golden_dir):
    g = _load(golden_dir, "mstgcn_small")
    ei = g["edge_index"].to(DEV)
    for name, c in g["cases"].items():
        m = MSTGCN(time_strides=c["time_strides"], **g["ctor"]).to(DEV)
        m.load_state_dict(c["state"])
        X = c["X"].to(DEV)
        with torch.no_grad():
            _close(m(X, ei), c["out"], 2e-4, 2e-5)               # two blocks of LayerNorm on GEMM rounding (= ASTGCN bar)
            _close(m(X, [ei] * 6), c["out_list"], 2e-4, 2e-5)    # per-timestep edge_index list path
        Xg = X.clone().requires_grad_(True)
        out = m(Xg, ei)
        _close(out, c["out"], 2e-4, 2e-5)
        _loss([out]).backward()
        _check_grads(m, c["grads"], 2e-3, 2e-5)
        _close(Xg.grad, c["gX"], 2e-3, 2e-5)


def test_dynamic_graph_signal_rebuilds_plans_on_device():
    """SURVEY 8f rank 4: a graph that changes per snapshot -> the layer's plan cache misses and the CSR operators are
    rebuilt on the device for each new edge list; piecewise-constant stretches (same array object) reuse the plan."""
    import numpy as np
    from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU
    from pytorch_geometric_temporal_b200.signal import DynamicGraphTemporalSignal
    rng = np.random.default_rng(0)
    n, T = 30, 6
    graphs = []
    for _ in range(3):
        pairs = {(int(a), int(b)) for a, b in rng.integers(0, n, (90, 2)) if a != b} | {(i, (i + 1) % n) for i in range(n)}
        ei = np.array(sorted(pairs)).T
        graphs.append((ei, rng.random(ei.shape[1]) * 0.9 + 0.1))
    order = [0, 0, 1, 1, 1, 2]                                   # piecewise-constant: 3 distinct graphs over 6 snapshots
    xs = [rng.standard_normal((n, 4)).astype(np.float32) for _ in range(T)]
    ys = [rng.standard_normal((n,)).astype(np.float32) for _ in range(T)]
    ds = DynamicGraphTemporalSignal([graphs[g][0] for g in order], [graphs[g][1] for g in order], xs, ys)
    torch.manual_seed(0)
    m = GConvGRU(4, 16, 3)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    mg = m.to(DEV)
    Hc = Hg = None
    builds = []
    for snap, dev_snap in zip(ds, ds.to(DEV)):
        Hc = R.gconv_gru_cell(sd, snap.x, snap.edge_index, snap.edge_attr, Hc)
        n0 = _lib.launch_count()
        with torch.no_grad():
            Hg = mg(dev_snap.x, dev_snap.edge_index, dev_snap.edge_attr, Hg)
        builds.append(_lib.launch_count() - n0)
        _close(Hg, Hc)
    # snapshots 1, 3, 4 reuse the previous snapshot's graph: no plan build, only the (K-1) SpMMs + gate kernels
    assert builds[1] < builds[0] and builds[3] < builds[2] and builds[4] == builds[3] and builds[5] > builds[4]


def test_mstgcn_distinct_graph_per_timestep(golden_dir):
    """per-timestep edge_index LIST with genuinely different graphs (mstgcn.py:96-115) against the oracle."""
    from oracle import attention as OA
    g = _load(golden_dir, "mstgcn_small")
    c = g["cases"]["s1"]
    base = g["edge_index"]
    gen = torch.Generator().manual_seed(5)
    eis = []
    for t in range(6):
        keep = torch.rand(base.size(1) // 2, generator=gen) > 0.25          # drop undirected pairs, keep symmetry
        und = {(int(a), int(b)) for a, b in base.t().tolist() if a < b}
        und = [p for p, k in zip(sorted(und), keep.tolist()) if k]
        ei = torch.tensor(sorted(und + [(b, a) for a, b in und]), dtype=torch.long).t().contiguous()
        eis.append(ei)
    want = OA.mstgcn(c["state"], c["X"], eis, g["ctor"]["nb_block"], 1)
    m = MSTGCN(time_strides=1, **g["ctor"]).to(DEV)
    m.load_state_dict(c["state"])
    with torch.no_grad():
        _close(m(c["X"].to(DEV), [e.to(DEV) for e in eis]), want, 2e-4, 2e-5)
