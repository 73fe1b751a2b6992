"""TGCN / TGCN2 training with a carried hidden state on the fused path: `stmp_tgcn_attn_fwd` with H forward, `stmp_tgcn_cell_bwd`
backward (k_tgcn_cell_bwd + k_tgcn_cell_bwd_reduce).  The loop of the reference's BatchedTGCN scripts and tgcn_example.py against the
unmodified reference (tests/golden/make_goldens_tgcn.py), and the fused path against the op-for-op autograd path
(`fused_training = False`)."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import TGCN, TGCN2
from tgcn_seq import load, model_for, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDENS = ["tgcn2_seq_metr_la_grads", "tgcn2_seq_pems_bay_grads", "tgcn_chickenpox_seq_grads"]


def _ran(before, name):
    return _lib.path_counters().get(name, 0) - before.get(name, 0)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got = got.detach().cpu()
    want = want.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _close_grad(got, want):
    _close(got, want, 1e-3, 1e-3 * want.abs().max().item() + 1e-6)


def _graph(seed=0):
    ei, ew, _ = synthetic.metr_la_like(seed, 16)
    return torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)


def _run_golden(g, fused):
    m = model_for(g, DEV, fused)
    H0 = g["H0"].to(DEV).requires_grad_(True) if "H0" in g else None
    c0 = _lib.path_counters()
    out, loss = run(m, g, DEV, H0)
    loss.backward()
    return m, H0, out, loss, c0


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", GOLDENS)
def test_carried_state_training_vs_reference_golden(golden_dir, name, fused):
    g = load(golden_dir, name)
    m, H0, out, loss, c0 = _run_golden(g, fused)
    steps = out.shape[0] if H0 is not None else out.shape[1]
    assert _ran(c0, "k_tgcn_cell_bwd") == ((steps - (H0 is None)) if fused else 0)
    _close(out, g["out"])
    _close(loss, g["loss"])
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        _close_grad(p.grad, g["grads"][k])
    if H0 is not None:
        _close_grad(H0.grad, g["gH0"])


def test_path_counters_of_a_fused_training_step(golden_dir):
    """A 12-step BatchedTGCN step: step 0 on the H = None pair, steps 1..11 on the cell backward, no SpMM anywhere."""
    g = load(golden_dir, "tgcn2_seq_metr_la_grads")
    _, _, _, _, c0 = _run_golden(g, True)
    assert {k: _ran(c0, k) for k in ("k_tgcn_cell_bwd", "k_tgcn_cell_bwd_reduce", "k_tgcn_attn_bwd", "k_tgcn_attn", "k_spmm")} == {
        "k_tgcn_cell_bwd": 11, "k_tgcn_cell_bwd_reduce": 11, "k_tgcn_attn_bwd": 1, "k_tgcn_attn": 12, "k_spmm": 0}


def _cell_case(cls, fin, improved=False, add_self_loops=True, B=3, seed=0):
    torch.manual_seed(seed)
    m = (TGCN(fin, 32, improved=improved, add_self_loops=add_self_loops) if cls is TGCN
         else TGCN2(fin, 32, B, improved=improved, add_self_loops=add_self_loops)).to(DEV)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn_like(p) * 0.1)
    lead = () if cls is TGCN else (B,)
    X = torch.randn(*lead, 207, fin, device=DEV)
    H = torch.randn(*lead, 207, 32, device=DEV) * 0.5
    w = torch.randn(*lead, 207, 32, device=DEV)
    return m, X, H, w


def test_training_forward_is_bit_equal_to_inference():
    ei, ew = _graph()
    m, X, H, _ = _cell_case(TGCN2, 2)
    c0 = _lib.path_counters()
    out = m(X, ei, ew, H)
    assert out.requires_grad and _ran(c0, "k_tgcn_attn") == 1
    with torch.no_grad():
        ref = m(X, ei, ew, H)
    assert torch.equal(out.detach(), ref)


def test_backward_is_deterministic():
    ei, ew = _graph()
    m, X, H, w = _cell_case(TGCN2, 4, B=16)

    def grads():
        m.zero_grad(set_to_none=True)
        Hl = H.clone().requires_grad_(True)
        (m(X, ei, ew, Hl) * w).sum().backward()
        return [Hl.grad] + [p.grad.clone() for p in m.parameters()]
    a, b = grads(), grads()
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("cls", [TGCN, TGCN2])
@pytest.mark.parametrize("fin", [1, 2, 3, 4])
def test_fused_cell_backward_vs_autograd(cls, fin):
    ei, ew = _graph(1)
    for improved in (False, True):
        for add_self_loops in (True, False):
            for h_grad in (True, False):
                m, X, H, w = _cell_case(cls, fin, improved, add_self_loops)
                res = []
                for fused in (True, False):
                    m.fused_training = fused
                    m.zero_grad(set_to_none=True)
                    Hl = H.clone().requires_grad_(h_grad)
                    c0 = _lib.path_counters()
                    out = m(X, ei, ew, Hl)
                    (out * w).sum().backward()
                    assert _ran(c0, "k_tgcn_cell_bwd") == int(fused)
                    res.append((out.detach(), Hl.grad, {k: p.grad.clone() for k, p in m.named_parameters()}))
                (of, hf, gf), (oa, ha, ga) = res
                _close(of, oa)
                assert (hf is None) == (not h_grad)
                if h_grad:
                    _close_grad(hf, ha)
                for k in ga:
                    _close_grad(gf[k], ga[k])


def test_routing_of_calls_outside_the_cell_backward():
    ei, ew = _graph()
    m, X, H, w = _cell_case(TGCN2, 2)
    c0 = _lib.path_counters()
    Xg = X.clone().requires_grad_(True)
    (m(Xg, ei, ew, H) * w).sum().backward()                               # gradient w.r.t. X
    assert Xg.grad is not None and Xg.grad.abs().max() > 0
    m16 = TGCN2(2, 16, 3).to(DEV)
    m16(X, ei, ew, H[..., :16]).sum().backward()                          # out_channels = 16
    m5 = TGCN2(5, 32, 3).to(DEV)
    X5 = torch.randn(3, 207, 5, device=DEV, requires_grad=True)
    m5(X5, ei, ew, H).sum().backward()                                    # in_channels = 5
    assert X5.grad is not None
    assert _ran(c0, "k_tgcn_cell_bwd") == 0
    # a non-contiguous state of the right shape is served by the fused path
    Hnc = torch.randn(3, 32, 207, device=DEV).transpose(1, 2).requires_grad_(True)
    assert not Hnc.is_contiguous()
    m.zero_grad(set_to_none=True)
    (m(X, ei, ew, Hnc) * w).sum().backward()
    assert _ran(c0, "k_tgcn_cell_bwd") == 1
    gf = [Hnc.grad.clone()] + [p.grad.clone() for p in m.parameters()]
    m.fused_training = False
    m.zero_grad(set_to_none=True)
    Hnc.grad = None
    (m(X, ei, ew, Hnc) * w).sum().backward()
    for a, b in zip(gf, [Hnc.grad] + [p.grad for p in m.parameters()]):
        _close_grad(a, b)


def test_unstaged_gather_on_a_50k_node_graph():
    """X[b] of 50 000 nodes x 4 features is 800 KB, beyond shared-memory staging: the global-memory gather serves the backward."""
    ei, ew = synthetic.large_graph(50000, 200000, seed=3)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    torch.manual_seed(2)
    m = TGCN2(4, 32, 2).to(DEV)
    X = torch.randn(2, 50000, 4, device=DEV)
    H = torch.randn(2, 50000, 32, device=DEV) * 0.5
    w = torch.randn(2, 50000, 32, device=DEV)
    res = []
    for fused in (True, False):
        m.fused_training = fused
        m.zero_grad(set_to_none=True)
        Hl = H.clone().requires_grad_(True)
        c0 = _lib.path_counters()
        out = m(X, ei, ew, Hl)
        (out * w).sum().backward()
        assert _ran(c0, "k_tgcn_cell_bwd") == int(fused)
        res.append([out.detach(), Hl.grad] + [p.grad.clone() for p in m.parameters()])
    _close(res[0][0], res[1][0])
    for a, b in zip(res[0][1:], res[1][1:]):
        _close_grad(a, b)


def test_cuda_graph_replay_of_a_training_step(golden_dir):
    g = load(golden_dir, "tgcn2_seq_pems_bay_grads")
    g = {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in g.items()}      # no host-to-device copy inside the capture
    m = model_for(g, DEV, True)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)
    state0 = {k: v.clone() for k, v in m.state_dict().items()}

    def step():
        opt.zero_grad(set_to_none=False)
        _, loss = run(m, g, DEV)
        loss.backward()
        opt.step()
        return loss

    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):                                                # warm-up on the capture stream (plans, Adam state)
            step()
    torch.cuda.current_stream().wait_stream(side)
    # the eager reference: two steps from the starting weights with a fresh optimizer
    m_e = model_for(g, DEV, True)
    m_e.load_state_dict(state0)
    opt_e = torch.optim.Adam(m_e.parameters(), lr=1e-3)
    eager_losses = []
    for _ in range(2):
        opt_e.zero_grad()
        _, le = run(m_e, g, DEV)
        le.backward()
        opt_e.step()
        eager_losses.append(le.detach())
    # the graph: restore the starting weights and a fresh optimizer state, capture one step and replay it twice
    m.load_state_dict(state0)
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step()
    m.load_state_dict(state0)
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    replay_losses = []
    for _ in range(2):
        graph.replay()
        replay_losses.append(loss.detach().clone())
    torch.cuda.synchronize()
    for a, b in zip(replay_losses, eager_losses):
        _close(a, b, 1e-5, 1e-7)
    for (k, p), pe in zip(m.named_parameters(), m_e.parameters()):
        _close(p, pe, 1e-5, 1e-6)


def test_abi_errors():
    ei, ew = _graph()
    m = TGCN2(2, 32, 1).to(DEV)
    plan = m._plan(ei, ew, 207)
    L = _lib.lib()
    buf = torch.zeros(1 << 20, device=DEV)
    p = _lib.ptr(buf)
    args = lambda B, fin, x: (plan.handle, B, fin, x, p, 207 * 32, p, p, p, p, p, p, p, p, p, None)
    assert L.stmp_tgcn_cell_bwd(*args(1, 5, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_cell_bwd(*args(1, 0, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_cell_bwd(*args(1, 2, None)) == _lib.STMP_EINVAL
    assert L.stmp_tgcn_cell_bwd(*args(65536, 2, p)) == _lib.STMP_ESHAPE
    assert L.stmp_tgcn_cell_bwd_workspace_bytes(plan.handle, 2) == 2 * 4 * (4 * 96 + 32 * 96 + 96) * 4     # 207 nodes: 4 CTAs per row
