"""GPU parity of the DCRNN family through the public modules (which call the C ABI): fused sequence
kernel and tiled path vs the CPU oracle and the committed reference goldens.
Tolerance (strict fp32 mode): rtol=1e-4, atol=1e-5 per layer output (SURVEY.md section 8d)."""
import os

import numpy as np

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN, BatchedDCRNN, DConv
from pytorch_geometric_temporal_b200.plan import GraphPlan

pytestmark = pytest.mark.gpu
DEV = "cuda"
RTOL, ATOL = 1e-4, 1e-5


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


def _close(got, want, rtol=RTOL, atol=ATOL):
    got = got.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def test_cfg2_batched_fused_vs_reference_golden(golden_dir):
    g = _load(golden_dir, "dcrnn_cfg2_batched")
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    m.load_state_dict(g["state"])
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    n0 = _lib.launch_count()
    with torch.no_grad():
        out = m(g["X"].to(DEV), ei, ew)
    assert _lib.launch_count() > n0  # the CUDA library really ran
    _close(out, g["out"])
    # second call hits the plan cache and the same kernel
    with torch.no_grad():
        _close(m(g["X"].to(DEV), ei, ew), g["out"])


def test_cfg2_batched_tiled_path_vs_golden(golden_dir):
    g = _load(golden_dir, "dcrnn_cfg2_batched")
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    m.load_state_dict(g["state"])
    out = m(g["X"].to(DEV), g["edge_index"].to(DEV), g["edge_weight"].to(DEV))  # grad enabled -> tiled path
    assert out.requires_grad
    _close(out, g["out"])


def test_cfg2_cell_vs_golden(golden_dir):
    g = _load(golden_dir, "dcrnn_cfg2_cell")
    m = DCRNN(2, 32, 2).to(DEV)
    m.load_state_dict(g["state"])
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    with torch.no_grad():
        _close(m(g["X"].to(DEV), ei, ew, g["H"].to(DEV)), g["out"])
        _close(m(g["X"].to(DEV), ei), g["out_noew_noh"])  # edge_weight=None, H=None
    _close(m(g["X"].to(DEV), ei, ew, g["H"].to(DEV)), g["out"])  # tiled


@pytest.mark.parametrize("K", [1, 3, 4])
def test_small_graph_K_fused_and_tiled_and_grads(golden_dir, K):
    g = _load(golden_dir, f"dcrnn_small_K{K}")
    m = DCRNN(3, 16, K).to(DEV)
    m.load_state_dict(g["state"])
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    with torch.no_grad():
        _close(m(g["X"].to(DEV), ei, ew, g["H"].to(DEV)), g["out"])  # fused
    X = g["X"].to(DEV).requires_grad_(True)
    H = g["H"].to(DEV).requires_grad_(True)
    out = m(X, ei, ew, H)  # tiled + autograd through the transposed SpMM
    _close(out, g["out"])
    w = torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)
    (out * w).sum().backward()
    _close(X.grad, g["gX"], 1e-3, 1e-5)
    _close(H.grad, g["gH"], 1e-3, 1e-5)
    for k, p in m.named_parameters():
        _close(p.grad, g["grads"][k], 1e-3, 1e-5)


def test_small_batched_K3(golden_dir):
    g = _load(golden_dir, "dcrnn_small_batched_K3")
    m = BatchedDCRNN(3, 16, 3).to(DEV)
    m.load_state_dict(g["state"])
    with torch.no_grad():
        _close(m(g["X"].to(DEV), g["edge_index"].to(DEV), g["edge_weight"].to(DEV)), g["out"])


@pytest.mark.parametrize("B", [1, 5, 300])
def test_fused_vs_oracle_many_windows_and_index_batching(B):
    """More windows than SMs (persistent loop + TMA double buffering) and the in-kernel window gather."""
    ei, ew, series = synthetic.metr_la_like(0, 400)
    ei_t, ew_t, s_t = torch.from_numpy(ei), torch.from_numpy(ew), torch.from_numpy(series)
    torch.manual_seed(B)
    m = BatchedDCRNN(2, 32, 2)
    starts = torch.randint(0, 400 - 12, (B,))
    X = torch.stack([s_t[s:s + 12] for s in starts.tolist()])
    nb = min(B, 4)  # oracle on a few windows only (seconds)
    want = R.batched_dcrnn(m.state_dict(), X[:nb], ei_t, ew_t)
    mg = m.to(DEV)
    with torch.no_grad():
        out = mg(X.to(DEV), ei_t.to(DEV), ew_t.to(DEV))
        out_idx = mg.forward_indexed(s_t.to(DEV), starts.to(DEV), 12, ei_t.to(DEV), ew_t.to(DEV))
    _close(out[:nb], want)
    assert torch.equal(out, out_idx)  # same kernel, X read in place from the resident series
    # windows are independent: permuting the batch permutes the output
    perm = torch.randperm(B)
    with torch.no_grad():
        assert torch.equal(mg(X[perm].to(DEV), ei_t.to(DEV), ew_t.to(DEV)), out[perm.to(DEV)])


def test_fused_recurrence_equals_chained_cells():
    """Size-independent property: T fused steps == T chained single-step calls with H carried."""
    ei, ew, series = synthetic.metr_la_like(0, 32)
    ei_t, ew_t = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    torch.manual_seed(0)
    mb = BatchedDCRNN(2, 32, 2).to(DEV)
    mc = DCRNN(2, 32, 2).to(DEV)
    mc.load_state_dict(mb.state_dict())
    X = torch.from_numpy(series[:12]).to(DEV)
    with torch.no_grad():
        seq = mb(X.unsqueeze(0), ei_t, ew_t)[0]
        H = None
        for t in range(12):
            H = mc(X[t], ei_t, ew_t, H)
            assert torch.allclose(H, seq[t], rtol=1e-5, atol=1e-6)


def test_dconv_layer_vs_oracle():
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    ei_t, ew_t = torch.from_numpy(ei), torch.from_numpy(ew)
    torch.manual_seed(3)
    conv = DConv(34, 32, 3)
    x = torch.randn(207, 34)
    want = R.dconv(x, R.dconv_operators(ei_t, ew_t, False, 207), conv.weight.detach(), conv.bias.detach())
    got = conv.to(DEV)(x.to(DEV), ei_t.to(DEV), ew_t.to(DEV))
    _close(got, want)


def test_unsupported_shapes_fall_back_to_tiled_not_cpu():
    ei, ew, _ = synthetic.pems_bay_like(0, 16)  # N=325 > 224 rows: fused kernel refuses
    ei_t, ew_t = torch.from_numpy(ei), torch.from_numpy(ew)
    torch.manual_seed(0)
    m = BatchedDCRNN(2, 32, 2)
    X = torch.randn(2, 3, 325, 2)
    want = R.batched_dcrnn(m.state_dict(), X, ei_t, ew_t)
    plan = GraphPlan(_lib.FLAVOR_DCONV, ei_t.to(DEV), ew_t.to(DEV), 325, flags=_lib.DCONV_ALLOW_DUPLICATES)
    assert not ops.dcrnn_seq_supported(plan, 2, 32, 2)
    n0 = _lib.launch_count()
    with torch.no_grad():
        got = m.to(DEV)(X.to(DEV), ei_t.to(DEV), ew_t.to(DEV))
    assert _lib.launch_count() > n0
    _close(got, want)


def test_full_bench_size_two_independent_kernels_agree():
    """Full BASELINE size (1184 windows x 12 steps, METR-LA shape): the wgmma kernel (fp16 hi/lo split operands, register accumulators)
    and the FFMA kernel (exact fp32, different thread mapping, TMA-staged inputs) are independent implementations of the
    same recurrence; they must agree to fp32 rounding on every one of the 94 M outputs, and a few windows are spot-checked
    against the oracle."""
    ei, ew, series = synthetic.metr_la_like(0, 4096)
    ei_t, ew_t, s_t = torch.from_numpy(ei), torch.from_numpy(ew), torch.from_numpy(series)
    torch.manual_seed(0)
    m = BatchedDCRNN(2, 32, 2)
    g = torch.Generator().manual_seed(1)
    starts = torch.randint(0, 4096 - 12, (1184,), generator=g)
    mg = BatchedDCRNN(2, 32, 2).to(DEV)
    mg.load_state_dict(m.state_dict())
    a = (s_t.to(DEV), starts.to(DEV), 12, ei_t.to(DEV), ew_t.to(DEV))
    try:
        with torch.no_grad():
            _lib.set_option("dcrnn_tc", 1)
            out_tc = mg.forward_indexed(*a)
            _lib.set_option("dcrnn_tc", 0)
            out_ff = mg.forward_indexed(*a)
    finally:
        _lib.set_option("dcrnn_tc", 1)
    assert out_tc.shape == (1184, 12, 207, 32)
    diff = (out_tc - out_ff).abs().max().item()
    assert diff < 2e-5, diff
    assert torch.isfinite(out_tc).all()
    pick = [0, 591, 1183]
    X = torch.stack([s_t[s:s + 12] for s in starts[pick].tolist()])
    want = R.batched_dcrnn(m.state_dict(), X, ei_t, ew_t)
    _close(out_tc[pick], want)
    _close(out_ff[pick], want)


def test_training_path_fused_forward_manual_backward_matches_autograd():
    """Training = fused forward (+ stash) and the hand-written reverse-time backward; gradients must match autograd
    through the tiled path (same module, `_fused_training` off) on the cfg2 shape."""
    ei, ew, series = synthetic.metr_la_like(0, 64)
    ei_t, ew_t = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    X = torch.from_numpy(series[:36]).reshape(3, 12, 207, 2).to(DEV)
    torch.manual_seed(0)
    a = BatchedDCRNN(2, 32, 2).to(DEV)
    b = BatchedDCRNN(2, 32, 2).to(DEV)
    b.load_state_dict(a.state_dict())
    b._fused_training = False
    w = torch.linspace(-1, 1, 3 * 12 * 207 * 32, device=DEV).view(3, 12, 207, 32)
    Xa, Xb = X.clone().requires_grad_(True), X.clone().requires_grad_(True)
    n0 = _lib.launch_count()
    oa = a(Xa, ei_t, ew_t)
    fused_fwd_launches = _lib.launch_count() - n0
    ob = b(Xb, ei_t, ew_t)
    assert fused_fwd_launches < 80 < _lib.launch_count() - n0 - fused_fwd_launches   # 1 fused launch (+ plan) vs the tiled graph
    _close(oa, ob.detach().cpu())
    (oa * w).sum().backward()
    (ob * w).sum().backward()
    _close(Xa.grad, Xb.grad.cpu(), 1e-3, 1e-5)
    for (k, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        _close(pa.grad, pb.grad.cpu(), 1e-3, 2e-4)


@pytest.mark.parametrize("fused_bwd", [True, False])
def test_training_backward_variants_cfg2(fused_bwd):
    """cfg2 shape, with an initial state and a window batch that is not a multiple of anything: the persistent backward
    kernel (stmp_dcrnn_bwd_basis + stmp_dcrnn_bwd_seq) and the per-step backward (stmp_gru_bwd_* + in-place transposed
    SpMM) must both reproduce autograd through the tiled path."""
    from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnSeqFn
    from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN
    ei, ew, series = synthetic.metr_la_like(3, 64)
    ei_t, ew_t = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    X = torch.from_numpy(series[:35]).reshape(5, 7, 207, 2).to(DEV)
    torch.manual_seed(1)
    a = BatchedDCRNN(2, 32, 2).to(DEV)
    b = BatchedDCRNN(2, 32, 2).to(DEV)
    b.load_state_dict(a.state_dict())
    b._fused_training = False
    w = torch.randn(5, 7, 207, 32, device=DEV)
    Xa, Xb = X.clone().requires_grad_(True), X.clone().requires_grad_(True)
    _DcrnnSeqFn.fused_backward = fused_bwd
    try:
        n0 = _lib.launch_count()
        oa = a(Xa, ei_t, ew_t)
        (oa * w).sum().backward()
        launches = _lib.launch_count() - n0
    finally:
        _DcrnnSeqFn.fused_backward = True
    (b(Xb, ei_t, ew_t) * w).sum().backward()
    if fused_bwd:
        assert launches <= 3 + 60                   # forward + basis + recurrence (+ one-time plan build)
    _close(Xa.grad, Xb.grad.cpu(), 1e-3, 1e-5)
    for (k, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        _close(pa.grad, pb.grad.cpu(), 1e-3, 2e-4)
    # single cell with an incoming state: gradient w.r.t. H flows through dh0
    c, d = DCRNN(2, 32, 2).to(DEV), DCRNN(2, 32, 2).to(DEV)
    d.load_state_dict(c.state_dict())
    d._fused_training = False
    x1 = torch.randn(207, 2, device=DEV)
    hc, hd = (torch.randn(207, 32, device=DEV) * 0.5).requires_grad_(True), None
    hd = hc.detach().clone().requires_grad_(True)
    _DcrnnSeqFn.fused_backward = fused_bwd
    try:
        (c(x1, ei_t, ew_t, hc) * w[0, 0]).sum().backward()
    finally:
        _DcrnnSeqFn.fused_backward = True
    (d(x1, ei_t, ew_t, hd) * w[0, 0]).sum().backward()
    _close(hc.grad, hd.grad.cpu(), 1e-3, 1e-5)
    for (k, pa), (_, pb) in zip(c.named_parameters(), d.named_parameters()):
        _close(pa.grad, pb.grad.cpu(), 1e-3, 1e-4)


def test_training_backward_general_K_small_graph():
    """K=3 / 16 hidden on a 40-node graph: fused FFMA forward with stash + the per-step backward (general K)."""
    import os
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "dcrnn_small_batched_K3.pt"), weights_only=False)
    ei, ew = g["edge_index"].to(DEV), g["edge_weight"].to(DEV)
    a, b = BatchedDCRNN(3, 16, 3).to(DEV), BatchedDCRNN(3, 16, 3).to(DEV)
    a.load_state_dict(g["state"]); b.load_state_dict(g["state"])
    b._fused_training = False
    Xa, Xb = g["X"].to(DEV).requires_grad_(True), g["X"].to(DEV).requires_grad_(True)
    oa, ob = a(Xa, ei, ew), b(Xb, ei, ew)
    _close(oa, g["out"]); _close(ob, g["out"])
    w = torch.randn_like(oa)
    (oa * w).sum().backward(); (ob * w).sum().backward()
    _close(Xa.grad, Xb.grad.cpu(), 1e-3, 1e-5)
    for (k, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        _close(pa.grad, pb.grad.cpu(), 1e-3, 1e-4)


@pytest.mark.parametrize("fused_bwd", [True, False])
def test_cfg2_training_gradients_vs_reference_golden(golden_dir, fused_bwd):
    """cfg2 shape: output and ALL gradients (input + parameters) of the fused forward + hand-written backward against the
    UNMODIFIED reference module's autograd (tests/golden/make_goldens_r2.py) -- not self-vs-self."""
    from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnSeqFn
    g = _load(golden_dir, "dcrnn_cfg2_grads")
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    m.load_state_dict(g["state"])
    X = g["X"].to(DEV).requires_grad_(True)
    before = _lib.path_counters()
    _DcrnnSeqFn.fused_backward = fused_bwd
    try:
        out = m(X, g["edge_index"].to(DEV), g["edge_weight"].to(DEV))
        w = torch.linspace(-1, 1, out.numel(), device=DEV).view_as(out)
        (out * w).sum().backward()
    finally:
        _DcrnnSeqFn.fused_backward = True
    after = _lib.path_counters()
    ran = {k for k, v in after.items() if v > before.get(k, 0)}
    assert "k_dcrnn_seq_tc" in ran                                     # the wgmma forward served the training call
    assert ("k_dcrnn_bwd_seq" in ran) == fused_bwd                     # and the persistent backward exactly when asked
    _close(out, g["out"])
    _close(X.grad, g["gX"], 1e-3, 1e-3 * g["gX"].abs().max().item())
    for k, p in m.named_parameters():
        ref = g["grads"][k]
        _close(p.grad, ref, 1e-3, 1e-3 * ref.abs().max().item())


def test_training_backward_with_permuted_input_requiring_grad():
    """X handed in as a dense non-contiguous view (B,N,F,T).permute(0,3,1,2) with requires_grad: dX must come back in X's
    index order (the kernels write dense (B,T,N,Cin) rows; a strided dX buffer would be scrambled)."""
    ei, ew, series = synthetic.metr_la_like(1, 64)
    ei_t, ew_t = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    base = torch.from_numpy(series[:24]).reshape(2, 12, 207, 2).to(DEV)
    torch.manual_seed(0)
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    w = torch.randn(2, 12, 207, 32, device=DEV)
    Xc = base.clone().requires_grad_(True)
    (m(Xc, ei_t, ew_t) * w).sum().backward()
    src = base.permute(0, 2, 3, 1).contiguous().requires_grad_(True)     # (B,N,F,T) storage
    Xp = src.permute(0, 3, 1, 2)                                         # (B,T,N,F) view, not contiguous
    assert not Xp.is_contiguous()
    m.zero_grad()
    (m(Xp, ei_t, ew_t) * w).sum().backward()
    _close(src.grad.permute(0, 3, 1, 2), Xc.grad.cpu(), 1e-5, 1e-6)


def test_path_counters_name_the_kernel_that_served_the_call():
    ei, ew, series = synthetic.metr_la_like(0, 32)
    ei_t, ew_t = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    X = torch.from_numpy(series[:24]).reshape(2, 12, 207, 2).to(DEV)
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    c0 = _lib.path_counters()
    with torch.no_grad():
        m(X, ei_t, ew_t)
    c1 = _lib.path_counters()
    assert c1.get("k_dcrnn_seq_tc", 0) == c0.get("k_dcrnn_seq_tc", 0) + 1
    m3 = BatchedDCRNN(2, 16, 3).to(DEV)                       # K=3 / 16 hidden: the FFMA sequence kernel
    with torch.no_grad():
        m3(X, ei_t, ew_t)
    c2 = _lib.path_counters()
    assert c2.get("k_dcrnn_seq", 0) == c1.get("k_dcrnn_seq", 0) + 1 and c2["k_dcrnn_seq_tc"] == c1["k_dcrnn_seq_tc"]


@pytest.mark.parametrize("cin", [1, 3, 4])
def test_training_persistent_backward_other_channel_counts(cin):
    """The persistent backward kernel pair for cin in {1, 3, 4} (scalar channel slots) against the per-step backward
    (stmp_gru_bwd_* + transposed SpMM), which is itself pinned to autograd and to the reference goldens."""
    from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnSeqFn
    ei, ew, _ = synthetic.metr_la_like(5, 16)
    ei_t, ew_t = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    torch.manual_seed(cin)
    X = torch.randn(4, 6, 207, cin, device=DEV)
    a, b = BatchedDCRNN(cin, 32, 2).to(DEV), BatchedDCRNN(cin, 32, 2).to(DEV)
    b.load_state_dict(a.state_dict())
    w = torch.randn(4, 6, 207, 32, device=DEV)
    Xa, Xb = X.clone().requires_grad_(True), X.clone().requires_grad_(True)
    c0 = _lib.path_counters()
    (a(Xa, ei_t, ew_t) * w).sum().backward()
    assert _lib.path_counters().get("k_dcrnn_bwd_seq", 0) == c0.get("k_dcrnn_bwd_seq", 0) + 1      # the persistent kernel served it
    _DcrnnSeqFn.fused_backward = False
    try:
        (b(Xb, ei_t, ew_t) * w).sum().backward()
    finally:
        _DcrnnSeqFn.fused_backward = True
    _close(Xa.grad, Xb.grad.cpu(), 1e-3, 1e-5)
    for (k, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        _close(pa.grad, pb.grad.cpu(), 1e-3, 2e-4)


@pytest.mark.parametrize("n_nodes,cin", [(207, 2), (50, 2), (121, 3)])
def test_persistent_backward_cluster_pair_equals_single_cta(n_nodes, cin):
    """Small batches run the reverse recurrence on a 2-CTA cluster per window (rows halved, dS exchanged through distributed shared
    memory); every row's arithmetic is the same sequence as in the one-CTA kernel, so the gradients must agree to the last bit."""
    rng = np.random.default_rng(n_nodes)
    E = 6 * n_nodes
    ring = np.arange(n_nodes)                      # every node keeps an in- and an out-edge (a zero degree is 1/0 in the DConv norms)
    src = np.concatenate([rng.integers(0, n_nodes, E), ring])
    dst = np.concatenate([rng.integers(0, n_nodes, E), (ring + 1) % n_nodes])
    ei = torch.from_numpy(np.stack([src, dst])).to(DEV)
    ew = torch.from_numpy((rng.random(E + n_nodes) + 0.1).astype(np.float32)).to(DEV)
    torch.manual_seed(cin + n_nodes)
    X = torch.randn(5, 6, n_nodes, cin, device=DEV)
    w = torch.randn(5, 6, n_nodes, 32, device=DEV)
    model = BatchedDCRNN(cin, 32, 2).to(DEV)
    grads = []
    for split in (1, 0):
        _lib.set_option("dcrnn_bwd_split", split)
        try:
            model.zero_grad()
            Xa = X.clone().requires_grad_(True)
            c0 = _lib.path_counters()
            (model(Xa, ei, ew) * w).sum().backward()
            c1 = _lib.path_counters()
        finally:
            _lib.set_option("dcrnn_bwd_split", 1)
        assert c1.get("k_dcrnn_bwd_seq", 0) == c0.get("k_dcrnn_bwd_seq", 0) + 1
        assert c1.get("k_dcrnn_bwd_seq[cluster2]", 0) - c0.get("k_dcrnn_bwd_seq[cluster2]", 0) == split
        grads.append([Xa.grad.clone()] + [p.grad.clone() for p in model.parameters()])
    for ga, gb in zip(*grads):
        assert bool(torch.isfinite(ga).all())
        assert torch.equal(ga, gb), f"max abs diff {(ga - gb).abs().max():.3e}"


@pytest.mark.parametrize("cin", [2, 1])
def test_forward_cluster_pair_equals_single_cta(cin):
    """Small batches may run the fused forward on a 2-CTA cluster per window (one MMA row tile each, H rows exchanged through distributed
    shared memory).  Row arithmetic is unchanged: outputs, the training stash and gradients agree with the one-CTA kernel to the last bit."""
    ei, ew, _ = synthetic.metr_la_like(4, 16)
    ei_t, ew_t = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    torch.manual_seed(10 + cin)
    X = torch.randn(7, 12, 207, cin, device=DEV)
    w = torch.randn(7, 12, 207, 32, device=DEV)
    model = BatchedDCRNN(cin, 32, 2).to(DEV)
    res = []
    for split in (1, 0):
        _lib.set_option("dcrnn_fwd_split", split)
        try:
            c0 = _lib.path_counters()
            with torch.no_grad():
                out = model(X, ei_t, ew_t)
            model.zero_grad()
            Xa = X.clone().requires_grad_(True)
            (model(Xa, ei_t, ew_t) * w).sum().backward()
            c1 = _lib.path_counters()
        finally:
            _lib.set_option("dcrnn_fwd_split", FWD_SPLIT_DEFAULT)
        assert c1.get("k_dcrnn_seq_tc[cluster2]", 0) - c0.get("k_dcrnn_seq_tc[cluster2]", 0) == 2 * split
        res.append([out, Xa.grad.clone()] + [p.grad.clone() for p in model.parameters()])
    for a, b in zip(*res):
        assert bool(torch.isfinite(a).all())
        assert torch.equal(a, b), f"max abs diff {(a - b).abs().max():.3e}"
    # one cell step with an incoming state (H0 is pushed into both gather buffers by the window prologue)
    cell = DCRNN(cin, 32, 2).to(DEV)
    x1, h1 = torch.randn(207, cin, device=DEV), torch.randn(207, 32, device=DEV) * 0.5
    outs = []
    for split in (1, 0):
        _lib.set_option("dcrnn_fwd_split", split)
        try:
            with torch.no_grad():
                outs.append(cell(x1, ei_t, ew_t, h1))
        finally:
            _lib.set_option("dcrnn_fwd_split", FWD_SPLIT_DEFAULT)
    assert torch.equal(outs[0], outs[1])


FWD_SPLIT_DEFAULT = 1
