"""Narrow-state DCRNN (cout <= 4): the reference's training model BatchedDCRNN(F, F, K=3) through the fused forward
(k_dcrnn_narrow_seq, served by stmp_dcrnn_seq_fwd) and the persistent backward (k_dcrnn_narrow_bwd)."""
import os

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN, BatchedDCRNN
from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnSeqFn
from pytorch_geometric_temporal_b200.plan import GraphPlan

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _grad_close(got, ref):
    _close(got, ref, 1e-3, 1e-3 * max(ref.abs().max().item(), 1e-12))


def _ran(before, after):
    """kernels launched between two path_counters() snapshots (the per-pack counters "<kernel>[pack P]" are left out)"""
    return {k for k, v in after.items() if v > before.get(k, 0) and "[pack " not in k}


class _Pack:
    """Pins the number of windows per CTA of the narrow kernels for a block (0 = automatic)."""

    def __init__(self, p):
        self.p = p

    def __enter__(self):
        _lib.set_option("dcrnn_narrow_pack", self.p)

    def __exit__(self, *exc):
        _lib.set_option("dcrnn_narrow_pack", 0)


def _random_graph(n, e, seed):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, n, (e,), generator=g)
    ring = torch.arange(n)
    ei = torch.stack([torch.cat([src, ring]), torch.cat([dst, (ring + 1) % n])])      # the ring keeps every degree > 0
    ew = torch.rand(ei.size(1), generator=g) + 0.1
    return ei, ew


def _model(cls, cin, cout, K, seed):
    torch.manual_seed(seed)
    m = cls(cin, cout, K)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith(".bias"):
                p.normal_(0, 0.1)
    return m


def _train(m, X, ei, ew, w):
    X = X.clone().requires_grad_(True)
    m.zero_grad()
    out = m(X, ei, ew)
    (out * w).sum().backward()
    return out.detach(), X.grad.clone(), [p.grad.clone() for p in m.parameters()]


# ---- goldens from the unmodified reference (tests/golden/make_goldens_narrow.py) -------------------------------------------
@pytest.mark.parametrize("name", ["dcrnn_narrow_pems_bay", "dcrnn_narrow_metr_la", "dcrnn_narrow_chickenpox"])
def test_batched_goldens_output_and_gradients(golden_dir, name):
    g = _load(golden_dir, name)
    F = g["F"]
    m = BatchedDCRNN(F, F, 3).to(DEV)
    m.load_state_dict(g["state"])
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    with torch.no_grad():
        m(g["X"].to(DEV), ei, ew)                                   # plan cached before the counters are read
    c0 = _lib.path_counters()
    with torch.no_grad():
        out = m(g["X"].to(DEV), ei, ew)
    c1 = _lib.path_counters()
    assert "k_dcrnn_narrow_seq" in _ran(c0, c1) and "k_spmm" not in _ran(c0, c1)
    _close(out, g["out"])
    X = g["X"].to(DEV).requires_grad_(True)
    out = m(X, ei, ew)
    c2 = _lib.path_counters()
    assert _ran(c1, c2) == {"k_dcrnn_narrow_seq"}                  # the training forward: one launch, no SpMM
    w = torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)
    (out * w).sum().backward()
    assert "k_dcrnn_narrow_bwd" in _ran(c2, _lib.path_counters())
    _close(out, g["out"])
    _grad_close(X.grad, g["gX"])
    for k, p in m.named_parameters():
        _grad_close(p.grad, g["grads"][k])


def test_cell_golden_with_incoming_state(golden_dir):
    g = _load(golden_dir, "dcrnn_narrow_cell")
    m = DCRNN(2, 2, 3).to(DEV)
    m.load_state_dict(g["state"])
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    with torch.no_grad():
        _close(m(g["X"].to(DEV), ei, ew, g["H"].to(DEV)), g["out"])
    X = g["X"].to(DEV).requires_grad_(True)
    H = g["H"].to(DEV).requires_grad_(True)
    c0 = _lib.path_counters()
    out = m(X, ei, ew, H)
    w = torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)
    (out * w).sum().backward()
    assert {"k_dcrnn_narrow_seq", "k_dcrnn_narrow_bwd"} <= _ran(c0, _lib.path_counters())
    _close(out, g["out"])
    _grad_close(X.grad, g["gX"])
    _grad_close(H.grad, g["gH"])
    for k, p in m.named_parameters():
        _grad_close(p.grad, g["grads"][k])


# ---- the whole envelope on a small random graph ---------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 3, 4])
@pytest.mark.parametrize("cout", [1, 2, 3, 4])
@pytest.mark.parametrize("cin", [1, 2, 3, 4])
def test_envelope_forward_vs_oracle_and_gradients_vs_both_backward_paths(cin, cout, K):
    ei, ew = _random_graph(23, 70, cin * 100 + cout * 10 + K)
    m = _model(BatchedDCRNN, cin, cout, K, K)
    X = torch.randn(3, 5, 23, cin, generator=torch.Generator().manual_seed(cin + 7 * cout))
    want = R.batched_dcrnn(m.state_dict(), X, ei, ew)
    m = m.to(DEV)
    Xd, eid, ewd = X.to(DEV), ei.to(DEV), ew.to(DEV)
    plan = GraphPlan(_lib.FLAVOR_DCONV, eid, ewd, 23, flags=_lib.DCONV_ALLOW_DUPLICATES)
    assert ops.dcrnn_seq_supported(plan, cin, cout, K) and ops.dcrnn_narrow_bwd_supported(plan, cin, cout, K)
    with torch.no_grad():
        _close(m(Xd, eid, ewd), want)
    w = torch.randn(3, 5, 23, cout, device=DEV)
    c0 = _lib.path_counters()
    out, gx, gp = _train(m, Xd, eid, ewd, w)
    assert "k_dcrnn_narrow_bwd" in _ran(c0, _lib.path_counters())
    _close(out, want)
    _DcrnnSeqFn.fused_backward = False
    try:
        _, gx_step, gp_step = _train(m, Xd, eid, ewd, w)
    finally:
        _DcrnnSeqFn.fused_backward = True
    m._fused_training = False
    try:
        _, gx_auto, gp_auto = _train(m, Xd, eid, ewd, w)
    finally:
        m._fused_training = True
    for ref_x, ref_p in ((gx_step, gp_step), (gx_auto, gp_auto)):
        _grad_close(gx, ref_x)
        for a, b in zip(gp, ref_p):
            _grad_close(a, b)


# ---- launch-shape invariance and determinism ------------------------------------------------------------------------------
def _effective_pack(requested, N, B):
    """The windows per CTA the library picks (choose_pack in dcrnn_narrow.cu): the requested P, or automatically B // SMs, clamped to
    1..8, then lowered to the thread capacity N * P <= 1024 (forward) / 512 (backward).  The shapes here are far from the
    shared-memory limit, so that one does not lower it."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    P = requested if requested > 0 else min(8, max(1, B // sms))
    return min(P, 1024 // N), min(P, 512 // N)


def _packs_ran(before, after):
    return {k for k, v in after.items() if v > before.get(k, 0) and "[pack " in k}


# (graph, cin, cout, K): on the 60-node graph P = 8 takes effect in both kernels (480 tasks: two per thread; P <= 4 runs one per
# thread), with CP = 4 and CP = 8 and K = 2..4; on PEMS-BAY a requested pack is lowered to the thread capacity.
@pytest.mark.parametrize("B", [64, 300])
@pytest.mark.parametrize("case", [("small", 2, 2, 3), ("small", 4, 4, 2), ("small", 1, 3, 4), ("pems_bay", 2, 2, 3)])
def test_pack_does_not_change_outputs_stash_or_gradients(case, B):
    graph, cin, cout, K = case
    if graph == "small":
        N, T = 60, 6
        ei, ew = _random_graph(N, 180, 11)
        s = torch.randn(120, N, cin, generator=torch.Generator().manual_seed(3))
    else:
        N, T = 325, 12
        ei, ew, series = synthetic.pems_bay_like(0, 120)
        ei, ew, s = torch.from_numpy(ei), torch.from_numpy(ew), torch.from_numpy(series)
    ei, ew, s = ei.to(DEV), ew.to(DEV), s.to(DEV)
    starts = torch.randint(0, 120 - T, (B,), generator=torch.Generator().manual_seed(B))
    X = torch.stack([s[i:i + T] for i in starts.tolist()])
    m = _model(BatchedDCRNN, cin, cout, K, 0).to(DEV)
    plan = m._plan(ei, ew, N)
    w = torch.randn(B, T, N, cout, device=DEV)
    results = []
    for P in (1, 2, 8, 0):
        with _Pack(P):
            c0 = _lib.path_counters()
            out, stash = ops.dcrnn_seq_fwd(plan, X, *m._params(), K, stash=True)
            results.append((out, stash) + _train(m, X, ei, ew, w))
            pf, pb = _effective_pack(P, N, B)
            assert _packs_ran(c0, _lib.path_counters()) == {f"k_dcrnn_narrow_seq[pack {pf}]", f"k_dcrnn_narrow_bwd[pack {pb}]"}
    if graph == "small":
        assert _effective_pack(8, N, B) == (8, 8)                  # the packed backward really runs with 8 windows per CTA
    ref = results[0]
    for r in results[1:]:
        assert torch.equal(r[0], ref[0]) and torch.equal(r[1], ref[1])
        assert torch.equal(r[2], ref[2]) and torch.equal(r[3], ref[3])
        assert all(torch.equal(a, b) for a, b in zip(r[4], ref[4]))
    again = _train(m, X, ei, ew, w)                                # run to run: bit-identical
    assert torch.equal(again[1], ref[3]) and all(torch.equal(a, b) for a, b in zip(again[2], ref[4]))


def test_forward_indexed_equals_materialised_windows_and_empty_calls():
    ei, ew, series = synthetic.metr_la_like(0, 500)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    s = torch.from_numpy(series).to(DEV)
    m = _model(BatchedDCRNN, 2, 2, 3, 1).to(DEV)
    starts = torch.randint(0, 500 - 12, (300,), generator=torch.Generator().manual_seed(0)).to(DEV)
    X = torch.stack([s[i:i + 12] for i in starts.tolist()])
    with torch.no_grad():
        a = m.forward_indexed(s, starts, 12, ei, ew)
        b = m(X, ei, ew)
        assert torch.equal(a, b)
        e0 = m.forward_indexed(s, starts[:0], 12, ei, ew)
        e1 = m(X[:, :0], ei, ew)
    assert e0.shape == (0, 12, 207, 2) and e1.shape == (300, 0, 207, 2)
    want = R.batched_dcrnn({k: v.cpu() for k, v in m.state_dict().items()}, X[:3].cpu(), ei.cpu(), ew.cpu())
    _close(a[:3], want)


# ---- edge cases -----------------------------------------------------------------------------------------------------------
def test_zero_degree_nodes_give_the_reference_non_finite_pattern():
    ei = torch.tensor([[0, 1, 2, 3], [1, 2, 3, 4]])   # path 0->1->2->3->4: node 0 has no in-edge, node 4 no out-edge
    x, h = torch.randn(5, 2), torch.randn(5, 2)
    m = _model(DCRNN, 2, 2, 3, 0)
    want = R.dcrnn_cell(m.state_dict(), x, ei, None, h)
    m = m.to(DEV)
    plan = m._plan(ei.to(DEV), None, 5)
    assert ops.dcrnn_seq_supported(plan, 2, 2, 3)
    for grad in (False, True):
        with torch.set_grad_enabled(grad):
            got = m(x.to(DEV), ei.to(DEV), None, h.to(DEV)).detach().cpu()
        assert torch.equal(torch.isfinite(got), torch.isfinite(want))
        fin = torch.isfinite(want)
        _close(got[fin], want[fin])


def test_graph_too_large_for_the_layout_takes_the_tiled_path():
    n = 1500
    ei, ew = _random_graph(n, 3000, 5)
    m = _model(BatchedDCRNN, 2, 2, 3, 2)
    X = torch.randn(2, 3, n, 2, generator=torch.Generator().manual_seed(1))
    want = R.batched_dcrnn(m.state_dict(), X, ei, ew)
    m = m.to(DEV)
    plan = m._plan(ei.to(DEV), ew.to(DEV), n)
    assert not ops.dcrnn_seq_supported(plan, 2, 2, 3)
    c0 = _lib.path_counters()
    with torch.no_grad():
        got = m(X.to(DEV), ei.to(DEV), ew.to(DEV))
    ran = _ran(c0, _lib.path_counters())
    assert "k_spmm" in ran and "k_dcrnn_narrow_seq" not in ran
    _close(got, want)


# ---- launches and CUDA graphs ---------------------------------------------------------------------------------------------
def test_training_step_launch_budget_at_the_pems_bay_shape():
    ei, ew, series = synthetic.pems_bay_like(0, 64)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    X = torch.from_numpy(series[:48]).reshape(4, 12, 325, 2).to(DEV).repeat(16, 1, 1, 1)        # B = 64
    m = _model(BatchedDCRNN, 2, 2, 3, 0).to(DEV)
    _train(m, X, ei, ew, torch.ones(64, 12, 325, 2, device=DEV))     # plan built, caches warm
    n0 = _lib.launch_count()
    out = m(X.requires_grad_(False), ei, ew)
    n1 = _lib.launch_count()
    assert n1 - n0 == 1                                            # the training forward is one library launch
    out.sum().backward()
    assert _lib.launch_count() - n0 <= 16


def test_cuda_graph_replay_gives_the_eager_gradients():
    ei, ew, series = synthetic.pems_bay_like(0, 64)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    X = torch.from_numpy(series[:48]).reshape(4, 12, 325, 2).to(DEV)
    m = _model(BatchedDCRNN, 2, 2, 3, 0).to(DEV)
    w = torch.randn(4, 12, 325, 2, device=DEV)

    def step():
        out = m(X, ei, ew)
        (out * w).sum().backward()

    for p in m.parameters():
        p.grad = None
    step()
    eager = [p.grad.clone() for p in m.parameters()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):                                         # warm-up on the capture stream
            for p in m.parameters():
                p.grad = None
            step()
    torch.cuda.current_stream().wait_stream(side)
    for p in m.parameters():
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for p in m.parameters():
        p.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for p, e in zip(m.parameters(), eager):
        assert torch.equal(p.grad, e)
