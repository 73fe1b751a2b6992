"""MPNNLSTM on the H100: every golden case against the float64 oracle (held to the reference's fingerprints by tests/test_mpnnlstm_cpu.py)
-- the training loop op for op with its eval pass on the row-split kernels, and the same calls under no_grad on the row-split kernels --,
the envelope and adversarial graphs against float64 in training and eval mode, BatchNorm's running statistics under no_grad, exact launch
counts, bit-reproducible calls, CUDA-graph replay, the routes that run op for op, the reference's unit test and the ABI's errors.
Tolerances are test_gpu_evolvegcn.py's (_close: the largest error over the float64 tensor's largest magnitude, 2e-4 for outputs, 1e-3
for gradients and running statistics)."""
import os

import pytest
import torch

from mpnnlstm_seq import Masks, graph_of, load, model_for, mpnn_forward, oracle_run, run
from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.nn.recurrent import MPNNLSTM
from pytorch_geometric_temporal_b200.plan import GraphPlan
from test_gpu_evolvegcn import _graph, ctypes_misaligned
from test_gpu_rows_envelope import _counted

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MP = ("k_mpnn_conv1", "k_mpnn_conv2", "k_mpnn_lstm")
BWD = {"k_mpnn_lstm_bwd": 1, "k_mpnn_bn_bwd": 2, "k_mpnn_conv2_bwd": 1, "k_mpnn_wgrad": 1, "k_mpnn_wgrad_reduce": 1}
ALL = MP + tuple(BWD) + ("k_mpnn_dx",)


@pytest.fixture(autouse=True)
def _fp32():
    """cuDNN's LSTM and cuBLAS in full fp32 on the op-for-op route."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _close(got, want, what, rtol=2e-4, scale=None):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = float((got - want).abs().max()) / ((float(want.abs().max()) if scale is None else scale) + 1e-30)
    assert err <= rtol, (what, err)


def _ran(c):
    return {k: v for k, v in c.items() if k in ALL}


def _want(fwd, train, dx=0):
    """The launches of `fwd` forward calls of which `train` run a backward (`dx` of them with dX)."""
    w = {k: fwd for k in MP}
    w.update({k: v * train for k, v in BWD.items()})
    w["k_mpnn_dx"] = dx
    return {k: v for k, v in w.items() if v}


def _dev(xy):
    return None if xy is None else (xy[0].to(DEV), xy[1].to(DEV))


def _bufs(m):
    return {k: v for k, v in m.state_dict().items() if "running" in k or "num_batches" in k}


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_golden_training_loop(name, fused):
    """The example's loop, fused (training calls on the row-split kernels and their backward) and with `fused_training = False` (training
    calls op for op); the eval pass (no_grad) runs on the row-split kernels either way."""
    c = load(GOLDEN)["cases"][name]
    ei, ew, train, ev = graph_of(c, GOLDEN)
    outs64, cost64, evs64, leaves, bufs64 = oracle_run(c, train, ev, ei, ew, c["epochs"])
    m = model_for(c, DEV)
    m.recurrent.fused_training = fused
    with _counted() as cnt:
        outs, cost, evs = run(m, _dev(train), _dev(ev), ei.to(DEV), None if ew is None else ew.to(DEV), c["epochs"], retain=True)
    calls, steps = 0 if ev is None else ev[0].shape[0], c["epochs"] * train[0].shape[0]
    assert _ran(cnt) == (_want(steps + calls, steps) if fused else _want(calls, 0)), cnt
    assert abs(float(cost.detach()) - float(cost64.detach())) <= 1e-5 * abs(float(cost64.detach()))
    _close(outs, outs64, "out")
    if evs64 is not None:
        _close(evs, evs64, "eval")
    for k, p in m.named_parameters():
        _close(p.grad, leaves[k].grad, k, 1e-3)
    for k, v in _bufs(m).items():
        if "num_batches" in k:
            assert int(v) == int(bufs64[k]), k
        else:
            _close(v, bufs64[k], k, 1e-3)


@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_golden_no_grad_training_mode(name):
    """The first epoch's calls under no_grad in training mode, on the row-split kernels: the same predictions (same masks) and the same
    running statistics as the float64 oracle's training loop."""
    c = load(GOLDEN)["cases"][name]
    if c["epochs"] != 1:
        pytest.skip("one epoch")
    ei, ew, train, _ = graph_of(c, GOLDEN)
    outs64, _, _, _, bufs64 = oracle_run(c, train, None, ei, ew, 1)
    m = model_for(c, DEV)
    X = train[0].to(DEV)
    with torch.no_grad(), _counted() as cnt:
        outs = torch.stack([m(x, ei.to(DEV), None if ew is None else ew.to(DEV)) for x in X])
    assert _ran(cnt) == {k: X.shape[0] for k in MP}, cnt
    _close(outs, outs64, "out")
    for k, v in _bufs(m).items():
        if "num_batches" in k:
            assert int(v) == int(bufs64[k]), k
        else:
            _close(v, bufs64[k], k, 1e-3)


def _model(cin, nodes, window, p, seed, momentum=0.1):
    torch.manual_seed(seed)
    m = MPNNLSTM(cin, 32, nodes, window, p)
    with torch.no_grad():
        for k, q in m.named_parameters():
            q.normal_(1.0 if "_batch_norm" in k and k.endswith("weight") else 0.0, 0.5)
        for bn in (m._batch_norm_1, m._batch_norm_2):
            bn.running_mean.normal_(0, 0.5)
            bn.running_var.uniform_(0.5, 2.0)
            bn.momentum = momentum
    m._masks = Masks(seed)
    m._uniforms = lambda R, dev: m._masks.draw(R).to(dev)
    return m.to(DEV)


def _check_grads(m, X, ei, ew, want_dx=True):
    """One training call with autograd on the row-split kernels and one backward against float64: output, dX, every parameter's gradient
    and the running statistics."""
    c = dict(window=m.window, nodes=m.num_nodes, cin=m.in_channels, p=m.dropout)
    P = {k: v.detach().double().cpu().requires_grad_(True) for k, v in m.named_parameters()}
    B = {k: (v.double() if v.is_floating_point() else v).cpu().clone() for k, v in m.named_buffers()}
    masks = Masks(0)
    masks.g.set_state(m._masks.g.get_state())
    u = masks.draw(X.size(0)).double() if m.training and m.dropout > 0 else None
    x64 = X.double().requires_grad_(want_dx)
    want = mpnn_forward(P, B, c, x64, ei, None if ew is None else ew.double(), u, m._batch_norm_1.training, m._batch_norm_1.momentum)
    coef = torch.randn(want.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    (want * coef).sum().backward()
    xd = X.to(DEV).requires_grad_(want_dx)
    m.zero_grad(set_to_none=True)
    with _counted() as cnt:
        got = m(xd, ei.to(DEV), None if ew is None else ew.to(DEV))
        (got * coef.float().to(DEV)).sum().backward()
    assert _ran(cnt) == _want(1, 1, int(want_dx)), cnt
    _close(got, want, "out")
    # BatchNorm with batch statistics cancels a constant shift of its input: where ReLU passes every row, the convolution bias's gradient
    # is exactly 0 and only rounding is left of it, so it is measured against the model's largest parameter gradient.
    top = max(float(g.grad.abs().max()) for g in P.values())
    for k, q in m.named_parameters():
        _close(q.grad, P[k].grad, k, 1e-3, top if (m._batch_norm_1.training and k.startswith("_convolution") and k.endswith("bias"))
               else None)
    if want_dx:
        _close(xd.grad, x64.grad, "dX", 1e-3)
    for k, v in m.named_buffers():
        if "num_batches" in k:
            assert int(v) == int(B[k]), k
        else:
            _close(v, B[k], k, 1e-3)


def _check_calls(m, X, ei, ew, calls=2, fused=True):
    """`calls` calls under no_grad in the model's mode against mpnn_forward in float64: outputs and the running statistics."""
    c = dict(window=m.window, nodes=m.num_nodes, cin=m.in_channels, p=m.dropout)
    P = {k: v.detach().double().cpu() for k, v in m.named_parameters()}
    B = {k: (v.double() if v.is_floating_point() else v).cpu().clone() for k, v in m.named_buffers()}
    masks = Masks(0)
    masks.g.set_state(m._masks.g.get_state())
    want = []
    for _ in range(calls):
        u = masks.draw(X.size(0)).double() if m.training and m.dropout > 0 else None
        want.append(mpnn_forward(P, B, c, X.double(), ei, None if ew is None else ew.double(), u, m._batch_norm_1.training,
                                 m._batch_norm_1.momentum))
    if not fused:
        m._fused_ok = lambda *a: False
    with torch.no_grad(), _counted() as cnt:
        got = [m(X.to(DEV), ei.to(DEV), None if ew is None else ew.to(DEV)) for _ in range(calls)]
    assert _ran(cnt) == (_want(calls, 0) if fused else {}), cnt
    for a, b in zip(got, want):
        _close(a, b, "out")
    for k, v in m.named_buffers():
        if "num_batches" in k:
            assert int(v) == int(B[k]), k
        else:
            _close(v, B[k], k, 1e-3)


@pytest.mark.parametrize("cin", [1, 4, 17, 32, 33, 64])
@pytest.mark.parametrize("window", [1, 2, 5])
@pytest.mark.parametrize("train", [True, False])
def test_envelope_against_float64(cin, window, train):
    for nodes, B in ((1, 2), (7, 1), (20, 3), (301, 2)):
        seed = 1000 * cin + 10 * window + nodes
        m = _model(cin, nodes, window, (0.5, 0.0)[seed % 2] if train else 0.5, seed, (0.1, None)[seed % 2])
        m.train(train)
        R = B * window * nodes
        ei, ew = _graph("holes" if seed % 3 == 1 else "random", R, seed)
        X = torch.randn(R, cin, generator=torch.Generator().manual_seed(seed))
        _check_calls(m, X, ei, ew if seed % 3 else None)
        if R > 2:                            # two-row batch statistics normalise every channel to +-1: what flows back is rounding
            _check_grads(m, X, ei, ew if seed % 3 else None, want_dx=seed % 2 == 0)


@pytest.mark.parametrize("grad", [True, False])
def test_frozen_batchnorm_in_training_mode(grad):
    """module.train() with both BatchNorms in eval mode (frozen statistics) and p > 0: dropout applies, BatchNorm uses and keeps its
    running statistics, as in the reference."""
    for cin, window, nodes in ((4, 1, 20), (33, 2, 7)):
        m = _model(cin, nodes, window, 0.5, 11 + cin)
        m.train()
        m._batch_norm_1.eval()
        m._batch_norm_2.eval()
        ei, ew = _graph("random", 2 * window * nodes, 11)
        X = torch.randn(2 * window * nodes, cin, generator=torch.Generator().manual_seed(11))
        if grad:
            _check_grads(m, X, ei, ew)
        else:
            _check_calls(m, X, ei, ew)


@pytest.mark.parametrize("train", [True, False])
def test_50000_rows_against_float64(train):
    m = _model(14, 50000, 1, 0.5, 7)
    m.train(train)
    ei, ew = _graph("random", 50000, 7)
    X = torch.randn(50000, 14, generator=torch.Generator().manual_seed(7))
    _check_calls(m, X, ei, ew, calls=1)
    _check_grads(m, X, ei, ew)


@pytest.mark.parametrize("kind", ["random", "holes", "E0"])
@pytest.mark.parametrize("fused", [True, False])
def test_adversarial_graphs(kind, fused):
    """Duplicates, self loops, rows without in-edges, isolated nodes, zero weights, and a graph without edges; both routes."""
    for train in (True, False):
        m = _model(4, 40, 2, 0.5, 3)
        m.train(train)
        ei, ew = _graph(kind, 160, 5)
        if kind == "random":
            ew[::4] = 0.0
        _check_calls(m, torch.randn(160, 4, generator=torch.Generator().manual_seed(5)), ei, ew, fused=fused)


def test_reproducible_and_modes():
    """Repeated no_grad calls are bit-identical in both modes; a training-mode call under no_grad updates the running statistics and
    num_batches_tracked, an eval-mode call leaves them alone."""
    ei, ew = _graph("random", 3000, 9)
    ei, ew = ei.to(DEV), ew.to(DEV)
    X = torch.randn(3000, 8, device=DEV)
    outs = {}
    for rep in range(2):
        m = _model(8, 1000, 3, 0.5, 9)
        with torch.no_grad():
            m.eval()
            before = {k: v.clone() for k, v in m.named_buffers()}
            e = m(X, ei, ew)
            assert all(torch.equal(v, before[k]) for k, v in m.named_buffers())
            m.train()
            t = m(X, ei, ew)
            assert int(m._batch_norm_1.num_batches_tracked) == 1 and int(m._batch_norm_2.num_batches_tracked) == 1
            assert not torch.equal(m._batch_norm_1.running_mean, before["_batch_norm_1.running_mean"])
        outs[rep] = (e, t, {k: v.clone() for k, v in m.named_buffers()})
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert all(torch.equal(v, outs[1][2][k]) for k, v in outs[0][2].items())


def test_cuda_graph_eval_call():
    m = _model(14, 50000, 1, 0.5, 2).eval()
    ei, ew = _graph("random", 50000, 2)
    ei, ew = ei.to(DEV), ew.to(DEV)
    X = torch.randn(50000, 14, device=DEV)
    with torch.no_grad():
        want = m(X, ei, ew)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(X, ei, ew)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            got = m(X, ei, ew)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_routes_op_for_op():
    """A gradient into edge_weight, float64 and hidden_size 64 run op for op (no row-split launch) and match float64."""
    ei, ew = _graph("random", 60, 3)
    X = torch.randn(60, 4, generator=torch.Generator().manual_seed(3))
    for dtype, hidden, grad in ((torch.float32, 32, True), (torch.float64, 32, False), (torch.float32, 64, False)):
        torch.manual_seed(3)
        m = MPNNLSTM(4, hidden, 20, 3, 0.0).to(DEV, dtype).eval()
        with torch.set_grad_enabled(grad), _counted() as cnt:
            out = m(X.to(DEV, dtype), ei.to(DEV), ew.to(DEV, dtype).requires_grad_(grad))
        assert _ran(cnt) == {}, cnt
        P = {k: v.detach().double().cpu() for k, v in m.named_parameters()}
        B = {k: (v.double() if v.is_floating_point() else v).cpu() for k, v in m.named_buffers()}
        if hidden == 32:
            want = mpnn_forward(P, B, dict(window=3, nodes=20, cin=4, p=0.0), X.double(), ei, ew.double(), None, False)
            _close(out, want, "out", 1e-4)
        else:
            assert out.shape == (20, 2 * 64 + 4 + 2)


def test_reference_unit_test():
    """test_mpnn_lstm_layer of the reference's test/recurrent_test.py, ported as written (a random graph for networkx's)."""
    number_of_nodes, edge_per_node, in_channels, hidden_size, window = 100, 10, 64, 32, 1
    g = torch.Generator().manual_seed(0)
    edge_index = torch.randint(0, number_of_nodes, (2, number_of_nodes * edge_per_node // 2), generator=g).to(DEV)
    X = (torch.rand(number_of_nodes, in_channels, generator=g) * 2 - 1).to(DEV)
    edge_weight = torch.rand(edge_index.size(1), generator=g).to(DEV)
    layer = MPNNLSTM(in_channels=in_channels, hidden_size=hidden_size, num_nodes=number_of_nodes, window=window, dropout=0.5).to(DEV)
    H = layer(X, edge_index, edge_weight)
    assert H.shape == (number_of_nodes, 2 * hidden_size + in_channels + window - 1)
    with torch.no_grad(), _counted() as cnt:
        H2 = layer(X, edge_index, edge_weight)
    assert H2.shape == H.shape and _ran(cnt) == {k: 1 for k in MP}


def test_abi_errors():
    ei, ew = _graph("random", 20, 1)
    ei, ew = ei.to(DEV), ew.to(DEV)
    L = _lib.lib()
    gcn = GraphPlan(_lib.FLAVOR_GCN, ei, ew, 20, None)
    improved = GraphPlan(_lib.FLAVOR_GCN, ei, ew, 20, None, flags=_lib.GCN_IMPROVED)
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei, ew, 20, "sym")
    assert L.stmp_mpnn_rows_supported(gcn.handle, 64, 32, 4) == 1 and L.stmp_mpnn_rows_supported(gcn.handle, 1, 32, 1) == 1
    assert L.stmp_mpnn_rows_supported(gcn.handle, 65, 32, 1) == 0 and L.stmp_mpnn_rows_supported(gcn.handle, 0, 32, 1) == 0
    assert L.stmp_mpnn_rows_supported(gcn.handle, 4, 64, 1) == 0 and L.stmp_mpnn_rows_supported(gcn.handle, 4, 32, 3) == 0
    assert L.stmp_mpnn_rows_supported(improved.handle, 4, 32, 1) == 0 and L.stmp_mpnn_rows_supported(cheb.handle, 4, 32, 1) == 0
    assert L.stmp_mpnn_rows_scratch_bytes(gcn.handle, 4, 32, 1) >= 3 * 20 * 32 * 4
    assert L.stmp_mpnn_rows_scratch_bytes(gcn.handle, 4, 64, 1) == 0
    buf = torch.zeros(1 << 20, device=DEV)
    p = _lib.ptr(buf)
    cnt = torch.zeros(2, dtype=torch.int64, device=DEV)
    c = _lib.ptr(cnt)

    def fwd(plan, cin=4, window=1, nodes=20, x=p, training=0, prob=0.0, u=None, count=c):
        return L.stmp_mpnn_rows_fwd(plan, cin, 32, window, nodes, x, p, p, p, p, p, p, p, p, count, 1e-5, 0.1, p, p, p, p, count, 1e-5,
                                    0.1, p, p, p, p, p, p, p, p, training, prob, u, p, None, p, None)
    assert fwd(None) == _lib.STMP_EINVAL
    assert fwd(cheb.handle) == _lib.STMP_EINVAL
    assert fwd(gcn.handle, cin=65) == _lib.STMP_EUNSUPPORTED
    assert fwd(improved.handle) == _lib.STMP_EUNSUPPORTED
    assert fwd(gcn.handle, x=None) == _lib.STMP_EINVAL
    assert fwd(gcn.handle, u=p) == _lib.STMP_EINVAL                          # dropout uniforms with p = 0
    assert fwd(gcn.handle, u=p, training=1, prob=1.0) == _lib.STMP_EINVAL    # ... and with p = 1
    one = GraphPlan(_lib.FLAVOR_GCN, torch.zeros(2, 0, dtype=torch.int64, device=DEV), None, 1, None)
    assert fwd(one.handle, nodes=1, training=1) == _lib.STMP_EINVAL          # one row in training mode
    assert L.stmp_mpnn_rows_bwd(gcn.handle, 4, 32, 1, 20, p, p, p, p, p, p, p, p, None, 1, 0.0, p, p, p, None, p, None) == _lib.STMP_EINVAL
    assert L.stmp_mpnn_rows_bwd(gcn.handle, 4, 32, 1, 20, *([p] * 9), 1, 1.0, p, p, p, None, p, None) == _lib.STMP_EINVAL
    assert L.stmp_mpnn_rows_wgrad(gcn.handle, 4, 32, 1, p, None, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_mpnn_rows_wgrad(gcn.handle, 4, 64, 1, p, p, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_mpnn_rows_workspace_bytes(gcn.handle, 4, 32, 1) > 0 and L.stmp_mpnn_rows_stash_bytes(gcn.handle, 4, 64, 1) == 0
    assert fwd(gcn.handle, nodes=3) == _lib.STMP_ESHAPE                      # 20 rows are not B x 1 x 3
    assert fwd(gcn.handle, x=ctypes_misaligned(buf)) == _lib.STMP_ESHAPE
    torch.cuda.synchronize()


def test_training_reproducible_equivariant_and_retain_graph():
    """The training forward equals the no_grad call bit for bit (same mode and masks); repeated backwards are bit-identical; gradients scale
    exactly with the loss (x8); a second backward through the retained graph gives the same gradients; fused against op for op."""
    ei, ew = _graph("random", 3000, 9)
    ei, ew = ei.to(DEV), ew.to(DEV)
    X = torch.randn(3000, 8, device=DEV)
    res = {}
    for fused in (True, False):
        grads = []
        for scale in (1.0, 1.0, 8.0):
            m = _model(8, 1000, 3, 0.5, 9)
            m.fused_training = fused
            with torch.no_grad():
                want = m(X, ei, ew)
            m = _model(8, 1000, 3, 0.5, 9)
            m.fused_training = fused
            Xg = X.clone().requires_grad_(True)
            out = m(Xg, ei, ew)
            if fused:
                assert torch.equal(out.detach(), want)
            loss = out.square().mean() * scale
            loss.backward(retain_graph=True)
            g1 = [q.grad.clone() for q in m.parameters()] + [Xg.grad.clone()]
            m.zero_grad()
            Xg.grad = None
            loss.backward()
            g2 = [q.grad.clone() for q in m.parameters()] + [Xg.grad.clone()]
            if fused:
                assert all(torch.equal(a, b) for a, b in zip(g1, g2))
            grads.append(g1)
        if fused:
            assert all(torch.equal(a, b) for a, b in zip(grads[0], grads[1]))
            assert all(torch.equal(a * 8, b) for a, b in zip(grads[0], grads[2]))
        res[fused] = grads[0]
    for a, b in zip(res[True], res[False]):
        _close(a, b, "grad", 1e-3)
