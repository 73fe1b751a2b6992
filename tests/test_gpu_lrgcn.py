"""LRGCN on the H100: the relational plans bit-exact against a CPU restatement, every golden case on the row-split cell and op for op against
the float64 oracle (held to the reference's fingerprints by tests/test_lrgcn_cpu.py), a float64 envelope over relations, bases, widths and
states, bit-equal training and inference forwards, launch counts, routing outside the envelope and the ABI's errors."""
import ctypes
import os

import pytest
import torch

from lrgcn_seq import edge_types, load, model_for, oracle_run, run, states_for
from gconvgru_seq import chickenpox_train_split
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import LRGCN
from pytorch_geometric_temporal_b200.plan import GraphPlan, RgcnPlan
from wikimaths_seq import load as load_wikimaths

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _plan_cpu(ei, rel, n, r):
    """(rowptr, col, val, eid) by destination and by source of relation r: entries in edge order per row, val = 1 / cnt_r(dst)."""
    idx = torch.nonzero(rel == r).flatten()
    src, dst = ei[0][idx], ei[1][idx]
    cnt = torch.bincount(dst, minlength=n).float()
    val = (1.0 / cnt[dst]) if idx.numel() else torch.zeros(0)
    out = []
    for key, other in ((dst, src), (src, dst)):
        order = torch.sort(key, stable=True).indices
        rowptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(torch.bincount(key, minlength=n), 0)])
        out.append((rowptr.int(), other[order].int(), val[order].float(), order.int()))
    return out


def _adversarial_graph(n, e, seed):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, max(1, n - 3), (e,), generator=g)        # the last nodes have no in-edge
    hub = torch.rand(e, generator=g) < 0.2
    dst[hub] = 0                                                    # a hub
    ei = torch.stack([src, dst])
    ei = torch.cat([ei, ei[:, :e // 8], torch.stack([src[:5], src[:5]])], 1)   # duplicates and self loops
    return ei


@pytest.mark.parametrize("n,e,types", [(20, 102, "src_lt_dst"), (300, 2000, "mixed"), (7, 0, "mixed"), (50, 200, "none")])
def test_plan_bit_exact(n, e, types):
    ei = _adversarial_graph(n, e, n) if e else torch.zeros(2, 0, dtype=torch.int64)
    E = ei.size(1)
    if types == "src_lt_dst":
        et = (ei[0] < ei[1]).long()
    elif types == "mixed":
        et = torch.arange(E) % 5 - 1                                 # -1 .. 3: relations 0, 1 and types that match neither
    else:
        et = torch.full((E,), 7)                                     # every relation empty
    for rel0, n_rel in ((0, 2), (1, 1), (2, 2)):
        plan = RgcnPlan(ei.to(DEV), et.to(DEV), n, rel0, n_rel)
        assert plan.n_ops == n_rel
        for k in range(n_rel):
            want = _plan_cpu(ei, et, n, rel0 + k)
            for t in (0, 1):
                got = [x.cpu() for x in plan.export(k, bool(t))]
                for a, b in zip(got, want[t]):
                    assert torch.equal(a, b)


def test_plan_rejects_bad_graphs():
    ei = torch.tensor([[0, 5], [1, 0]], device=DEV)
    with pytest.raises(RuntimeError, match="outside"):
        RgcnPlan(ei, torch.zeros(2, dtype=torch.int64, device=DEV), 3, 0, 1)
    out = ctypes.c_void_p()
    L = _lib.lib()
    assert L.stmp_plan_create_rgcn(3, 1, _lib.ptr(ei), _lib.ptr(ei), 0, 3, None, ctypes.byref(out)) == _lib.STMP_EINVAL
    assert L.stmp_plan_create_rgcn(3, 1, _lib.ptr(ei), None, 0, 1, None, ctypes.byref(out)) == _lib.STMP_EINVAL
    assert L.stmp_plan_create(_lib.FLAVOR_RGCN, 3, 1, _lib.ptr(ei), None, 0, -1.0, 0, None, ctypes.byref(out)) == _lib.STMP_EINVAL


def _graph(c):
    if c["graph"] == "chickenpox":
        return chickenpox_train_split()
    w = load_wikimaths(GOLDEN)
    return w["edge_index"], w["edge_weight"], w["X"], w["Y"]


def _close(got, want, what, rtol=2e-4):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    scale = float(want.abs().max()) + 1e-30
    err = float((got - want).abs().max()) / scale
    assert err <= rtol, (what, err)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_golden_cases(name, fused):
    c = load(GOLDEN)["cases"][name]
    ei, ew, X, Y = _graph(c)
    et = edge_types(c["types"], ei, ew)
    H0, C0 = states_for(c, X.shape[1], dtype=torch.float64)
    outs64, cost64, leaves = oracle_run(c, X, Y, ei, et, H0, C0)
    cost64.backward()
    m = model_for(c, DEV, fused)
    h0, c0 = states_for(c, X.shape[1], DEV)
    outs, cost = run(m, X.to(DEV), Y.to(DEV), ei.to(DEV), et.to(DEV), h0, c0)
    cost.backward()
    assert abs(float(cost.detach()) - float(cost64.detach())) <= 1e-5 * abs(float(cost64.detach()))
    _close(outs, outs64, "out")
    for k, p in m.named_parameters():
        ref = leaves[k].grad
        if float(ref.abs().max()) == 0:                # structural zeros: the tutorial's relation weights
            assert float(p.grad.abs().max()) == 0, k
        else:
            _close(p.grad, ref, k, 1e-3)
    if H0 is not None:
        _close(h0.grad, H0.grad, "gH0", 1e-3)
        _close(c0.grad, C0.grad, "gC0", 1e-3)


def _envelope_case(n, cin, co, R, B, with_state, seed):
    g = torch.Generator().manual_seed(seed)
    e = 4 * n
    ei = _adversarial_graph(n, e, seed) if n > 3 else torch.randint(0, n, (2, e), generator=g)
    et = torch.randint(0, R + 1, (ei.size(1),), generator=g)        # type R matches no relation
    torch.manual_seed(seed)
    m = LRGCN(cin, co, R, B)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.3)
    X = torch.randn(n, cin, generator=g)
    H = torch.randn(n, co, generator=g) * 0.5 if with_state else None
    C = torch.randn(n, co, generator=g) * 0.5 if with_state else None
    return m, ei, et, X, H, C


@pytest.mark.parametrize("R,B,co", [(1, None, 32), (1, 1, 32), (2, None, 32), (2, 1, 32), (2, 2, 32), (1, None, 64), (1, 2, 64)])
@pytest.mark.parametrize("cin", [1, 5, 16])
@pytest.mark.parametrize("n,with_state", [(1, True), (37, False), (1068, True), (50000, True)])
def test_envelope_against_float64(R, B, co, cin, n, with_state):
    m, ei, et, X, H, C = _envelope_case(n, cin, co, R, B, with_state, n + cin + 7 * R)
    m64 = LRGCN(cin, co, R, B).double()
    m64.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    leaves = [t.double().requires_grad_(True) if t is not None else None for t in (X, H, C)]
    p = {k: v for k, v in m64.state_dict(keep_vars=True).items()}
    from lrgcn_seq import lrgcn_cell
    z = torch.zeros(n, co, dtype=torch.float64)
    h64, c64 = lrgcn_cell(p, leaves[0], ei, et, leaves[1] if with_state else z, leaves[2] if with_state else z, R)
    gh, gc = torch.randn(n, co, dtype=torch.float64) * 0.1, torch.randn(n, co, dtype=torch.float64) * 0.1
    (h64 * gh).sum().add_((c64 * gc).sum()).backward()
    md = m.to(DEV)
    xs = [t.to(DEV).requires_grad_(True) if t is not None else None for t in (X, H, C)]
    n0 = _lib.path_counters().get("k_lstm_rows_fwd", 0) + _lib.path_counters().get("k_lstm_wide_rows_fwd", 0)
    h, c = md(xs[0], ei.to(DEV), et.to(DEV), xs[1], xs[2])
    n1 = _lib.path_counters().get("k_lstm_rows_fwd", 0) + _lib.path_counters().get("k_lstm_wide_rows_fwd", 0)
    assert n1 == n0 + 1                                   # inside the envelope: the row-split cell served it
    (h * gh.float().to(DEV)).sum().add_((c * gc.float().to(DEV)).sum()).backward()
    _close(h, h64, "H", 1e-4)
    _close(c, c64, "C", 1e-4)
    for k, q in md.named_parameters():
        _close(q.grad, p[k].grad, k, 1e-3)
    for t, ref, name in zip(xs, leaves, ("dX", "dH", "dC")):
        if t is not None:
            _close(t.grad, ref.grad, name, 1e-3)


@pytest.mark.parametrize("R,co", [(2, 32), (1, 64)])
def test_training_forward_equals_inference_and_repeats(R, co):
    m, ei, et, X, H, C = _envelope_case(700, 5, co, R, 2, True, 3)
    m = m.to(DEV)
    args = (X.to(DEV), ei.to(DEV), et.to(DEV), H.to(DEV), C.to(DEV))
    with torch.no_grad():
        hi, ci = m(*args)
    n0 = _lib.launch_count()
    with torch.no_grad():
        m(*args)
    assert _lib.launch_count() - n0 == 1                  # after the pack: one launch per step
    h, c = m(*args)
    assert torch.equal(h, hi) and torch.equal(c, ci)
    grads = []
    for scale in (1.0, 1.0, 8.0):
        m.zero_grad()
        h, c = m(*args)
        ((h.square().mean() + c.mean()) * scale).backward()
        grads.append([p.grad.clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(grads[0], grads[1]))
    assert all(torch.equal(a * 8, b) for a, b in zip(grads[0], grads[2]))


@pytest.mark.parametrize("cin,co,R", [(4, 32, 3), (4, 48, 1), (17, 32, 2), (4, 64, 2)])
def test_outside_the_envelope_runs_op_for_op(cin, co, R):
    m, ei, et, X, H, C = _envelope_case(200, cin, co, R, None, True, 5)
    m64 = LRGCN(cin, co, R, None).double()
    m64.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    from lrgcn_seq import lrgcn_cell
    h64, c64 = lrgcn_cell(m64.state_dict(), X.double(), ei, et, H.double(), C.double(), R)
    md = m.to(DEV)
    before = dict(_lib.path_counters())
    with torch.no_grad():
        h, c = md(X.to(DEV), ei.to(DEV), et.to(DEV), H.to(DEV), C.to(DEV))
    after = _lib.path_counters()
    assert all(after.get(k, 0) == before.get(k, 0) for k in ("k_lstm_rows_fwd", "k_lstm_wide_rows_fwd"))
    _close(h, h64, "H", 1e-4)
    _close(c, c64, "C", 1e-4)


def test_cuda_graph_tutorial_epoch():
    c = load(GOLDEN)["cases"]["tutorial"]
    ei, ew, X, Y = chickenpox_train_split()
    m = model_for(c, DEV)
    X, Y, ei, ew = X.to(DEV), Y.to(DEV), ei.to(DEV), ew.to(DEV)
    with torch.no_grad():
        want, _ = run(m, X, Y, ei, ew)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        run(m, X, Y, ei, ew)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.no_grad():
        got, _ = run(m, X, Y, ei, ew)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_abi_errors():
    ei, ew, _, _ = chickenpox_train_split()
    L = _lib.lib()
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 20, "sym")
    two = RgcnPlan(ei.to(DEV), (ei[0] < ei[1]).long().to(DEV), 20, 0, 2)
    GCV, GC = _lib.LSTM_GCONV, _lib.LSTM_GC
    assert L.stmp_lstm_rows_supported(two.handle, GCV, 2, 16, 32) == 1
    assert L.stmp_lstm_rows_supported(two.handle, GCV, 2, 16, 64) == 0
    assert L.stmp_lstm_rows_supported(two.handle, GC, 2, 4, 32) == 0
    assert L.stmp_lstm_rows_supported(two.handle, GCV, 2, 17, 32) == 0
    assert L.stmp_lstm_rows_supported(cheb.handle, GCV, 2, 4, 32) == 0
    buf = torch.zeros(1 << 20, device=DEV)
    p = _lib.ptr(buf)
    ld = ops.lstm_rows_basis_ld(GCV, 2, 4)
    assert ld == 112 and ops.lstm_rows_basis_ld(GCV, 2, 16) == 144
    fwd = lambda plan, co_entry: getattr(L, co_entry)(plan.handle, GCV, 2, 4, p, p, p, p, p, None, p, p, p, p, ld, None)
    assert fwd(cheb, "stmp_lstm_rows_fwd") == _lib.STMP_EUNSUPPORTED
    assert fwd(two, "stmp_lstm_wide_rows_fwd") == _lib.STMP_EUNSUPPORTED
    assert L.stmp_lstm_rows_bwd(cheb.handle, GCV, 2, 4, p, p, p, p, p, p, None, p, p, p, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_lstm_wide_rows_pack_weights(GCV, 2, 4, p, p, None, None, p, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_lstm_rows_wgrad2(17, 20, ld, p, p, p, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_lstm_rows_wgrad2(4, 20, ld + 8, p, p, p, p, p, None) == _lib.STMP_ESHAPE
    assert L.stmp_lstm_rows_wgrad2(4, 20, ld, None, p, p, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_lstm_rows_wgrad2_workspace_bytes(16) > 0 and L.stmp_lstm_rows_wgrad2_workspace_bytes(17) == 0
    assert L.stmp_lstm_rows_scratch_bytes(two.handle) == (20 * 96 + 2 * 96) * 4
    torch.cuda.synchronize()
