"""MTGNN on the H100: every golden case on both routes (the fused graph kernels and op for op), in train and eval mode, against the
reference's float64 values; the graph build, the propagation and their backward against float64 across the envelope (node counts
1..4 096, k 1..64 and k = N, embedding widths 1..64, depths 1..4, channels 1..64, steps 1..181, B = 0..64, every gradient subset, a hub
column, empty columns, a full and a partly empty predefined A); the tie rule on saturated rows; a training forward bit-equal to the
no_grad call, repeatable backwards and loss-scale equivariance; exact launch counts; CUDA-graph replay of a training step; the routes
outside the envelope and the ABI's errors.

The criterion, per tensor (DESIGN §5): the fused route's largest error against float64 is at most 4 times the float32 op-for-op route's
plus 2^-20 of the tensor's largest float64 magnitude.  The goldens are held to it through their fingerprints (four fixed projections and
the norm), with the norm as the scale."""
import ctypes
import os

import pytest
import torch

from mtgnn_seq import CASES, fingerprint, inputs, load, model_for, run
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.attention import MTGNN
from pytorch_geometric_temporal_b200.nn.attention import mtgnn as M
from test_gpu_rows_envelope import _counted

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
D = torch.float64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GRAPH = ("k_mtgnn_topk", "k_mtgnn_col_count", "k_mtgnn_col_scan", "k_mtgnn_col_fill")
ALL = GRAPH + ("k_mtgnn_dense_rows", "k_mtgnn_hop", "k_mtgnn_hop_adjoint", "k_mtgnn_dvals", "k_mtgnn_graph_dd", "k_mtgnn_graph_dm")


@pytest.fixture(autouse=True)
def _fp32():
    """cuBLAS in full fp32 on the op-for-op route."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _ran(c):
    return {k: v for k, v in c.items() if k in ALL}


def _criterion(fused, op, want, what, scale=None):
    fused, op, want = (t.detach().double().cpu() for t in (fused, op, want))
    assert fused.shape == want.shape == op.shape, (what, fused.shape, want.shape)
    if want.numel() == 0:
        return
    scale = float(want.abs().max()) if scale is None else scale
    ef, eo = float((fused - want).abs().max()), float((op - want).abs().max())
    assert ef <= 4 * eo + 2.0 ** -20 * scale, (what, ef, eo, scale)


def _run_route(c, fused):
    m = model_for(c, MTGNN, DEV, torch.float32)
    m.fused_training = fused
    with _counted() as cnt:
        got = run(m, c, DEV, torch.float32)
    torch.cuda.synchronize()
    return got, _ran(cnt)


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_both_routes(name):
    c = load(GOLDEN)["cases"][name]
    gf, ran_f = _run_route(CASES[name], True)
    go, ran_o = _run_route(CASES[name], False)
    model = CASES[name]["model"]
    if model["gcn_true"]:
        L, depth = model["layers"], model["gcn_depth"]
        # training steps run fused only on the fused route; the eval call (no_grad) runs fused on both
        assert ran_f.get("k_mtgnn_hop_adjoint") == 2 * depth * L * 2, ran_f
        assert ran_f.get("k_mtgnn_hop") == 2 * depth * L * 3, ran_f
        assert "k_mtgnn_hop_adjoint" not in ran_o and ran_o.get("k_mtgnn_hop") == 2 * depth * L, ran_o
    else:
        assert not ran_f and not ran_o
    assert set(gf) == set(c["fingerprints"])
    for k, fp in c["fingerprints"].items():
        _criterion(fingerprint(gf[k]), fingerprint(go[k]), fp, k, scale=float(fp[-1]))


# ---- the kernels against float64 ------------------------------------------------------------------------------------------------
def _dense_from(pattern, vals, n, w):
    """(S1, S2) as dense float64 matrices from the kernels' structures."""
    pattern, vals = pattern.cpu().long(), vals.detach().cpu().double()
    nw = n * w
    col1, cnt1 = pattern[:nw].view(n, w), pattern[nw:nw + n]
    v1, v2, g1, g2 = vals[:nw].view(n, w), vals[nw:2 * nw].view(n, w), vals[2 * nw:2 * nw + n], vals[2 * nw + n:]
    S1, S2 = torch.diag(g1), torch.diag(g2)
    for i in range(n):
        c = int(cnt1[i])
        S1[i, col1[i, :c]] += v1[i, :c]
        S2[col1[i, :c], i] += v2[i, :c]
    return S1, S2


def _defined(pattern, n, w):
    """The pattern without the unused tail of the column arrays (capacity N w, of which ptr2[N] entries are used)."""
    nw = n * w
    nnz = int(pattern[nw + 2 * n])
    row2 = pattern[nw + 2 * n + 1:]
    return torch.cat((pattern[:nw + 2 * n + 1], row2[:nnz], row2[nw:nw + nnz]))


def _graph_dense(m1, m2, k, talpha):
    """The reference's graph and both normalised operators, in m1's dtype."""
    a = m1 @ m2.T - m2 @ m1.T
    A = torch.relu(torch.tanh(talpha * a))
    mask = torch.zeros_like(A).scatter_(1, A.topk(k, 1).indices, 1.0)
    A = A * mask
    eye = torch.eye(A.shape[0], dtype=A.dtype, device=A.device)
    S1, S2 = A + eye, A.T + eye
    return A, S1 / S1.sum(1).view(-1, 1), S2 / S2.sum(1).view(-1, 1)


def _gap_ok(m1, m2, k, talpha):
    m1, m2 = m1.double().cpu(), m2.double().cpu()
    a = m1 @ m2.T - m2 @ m1.T
    A = torch.relu(torch.tanh(talpha * a))
    if k >= A.shape[1]:
        return torch.ones(A.shape[0], dtype=torch.bool)
    top = A.topk(k + 1, 1).values
    return (top[:, k - 1] <= 0) | ((top[:, k - 1] - top[:, k]) > 2.0 ** -20 * top[:, k - 1])


def _embeddings(n, dim, seed, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.tanh(scale * torch.randn(n, dim, generator=g)).to(DEV), torch.tanh(scale * torch.randn(n, dim, generator=g)).to(DEV))


@pytest.mark.parametrize("n,k,dim", [(1, 1, 1), (2, 1, 40), (2, 2, 64), (20, 20, 1), (20, 20, 40), (21, 20, 40), (31, 30, 64),
                                     (65, 64, 1), (207, 1, 1), (207, 20, 40), (207, 64, 64), (325, 30, 40), (325, 20, 1),
                                     (862, 1, 40), (862, 20, 64), (862, 30, 1), (862, 64, 40), (4096, 64, 64), (4096, 20, 40),
                                     (4096, 1, 1), (64, 64, 8), (300, 64, 40)])
def test_graph_build_against_float64(n, k, dim):
    talpha = 3.0
    m1, m2 = _embeddings(n, dim, n * 7 + k, scale=0.3 / max(1.0, dim ** 0.5 / 4))
    ok = _gap_ok(m1, m2, k, talpha)             # near-tie rows screened: float32 may pick another member of the tie
    pattern, state, vals = ops.mtgnn_graph_fwd(m1, m2, k, talpha)
    S1, S2 = _dense_from(pattern, vals, n, k)
    _, W1, W2 = _graph_dense(m1.double().cpu(), m2.double().cpu(), k, talpha)
    _, O1, O2 = _graph_dense(m1, m2, k, talpha)
    rows = ok.nonzero().flatten()
    assert rows.numel() >= 0.9 * n
    _criterion(S1[rows], O1.cpu()[rows], W1[rows], "S1")
    if bool(ok.all()):                          # a column of operator 2 depends on every row's selection
        _criterion(S2, O2.cpu(), W2, "S2")
    p = pattern.cpu()
    nw = n * k
    cnt1, ptr2 = p[nw:nw + n], p[nw + n:nw + 2 * n + 1]
    assert int(ptr2[-1]) == int(cnt1.sum()) and bool((cnt1 <= k).all())
    again = ops.mtgnn_graph_fwd(m1, m2, k, talpha)
    assert torch.equal(_defined(pattern, n, k), _defined(again[0], n, k))
    assert torch.equal(state, again[1]) and torch.equal(vals, again[2])


def test_tie_rule_on_saturated_rows(capsys):
    """tanh rounds to 1.0 in float32 once |alpha z| > 9: with large embeddings most positive entries of a row are exactly 1.0.  Among
    equal values the kernel keeps the lower columns.  torch.topk on CUDA is compared at the reference's shape and the agreement printed
    (torch documents no order among ties)."""
    n, k, dim, talpha = 207, 20, 40, 3.0
    m1, m2 = _embeddings(n, dim, 11, scale=5.0)
    pattern, _, _ = ops.mtgnn_graph_fwd(m1, m2, k, talpha)
    p = pattern.cpu()
    col1, cnt1 = p[:n * k].view(n, k).long(), p[n * k:n * k + n]
    a = m1 @ m2.T - m2 @ m1.T
    A = torch.relu(torch.tanh(talpha * a))
    saturated = 0
    agree = 0
    for i in range(n):
        ones = (A[i] == 1.0).nonzero().flatten().cpu()
        if ones.numel() <= k:
            continue
        saturated += 1
        got = set(col1[i, :int(cnt1[i])].tolist())
        assert got == set(ones[:k].tolist()), i          # the k lowest columns among the equal values
        agree += got == set(A[i].topk(k).indices.cpu().tolist())
    assert saturated > n // 2
    with capsys.disabled():
        print(f"\n[mtgnn tie rule] saturated rows {saturated}, torch.topk on CUDA picks the same set in {agree}")


def _prop_case(B, C, n, T, k, depth, dim, seed, predefined=None):
    g = torch.Generator().manual_seed(seed)
    alpha, talpha, Co = 0.05, 3.0, 6
    X = torch.randn(B, C, n, T, generator=g)
    W1 = 0.3 * torch.randn(Co, (depth + 1) * C, 1, 1, generator=g)
    W2 = 0.3 * torch.randn(Co, (depth + 1) * C, 1, 1, generator=g)
    b1, b2 = torch.randn(Co, generator=g), torch.randn(Co, generator=g)
    gy = torch.randn(B, Co, n, T, generator=g)
    m1, m2 = _embeddings(n, dim, seed + 1, scale=0.3 / max(1.0, dim ** 0.5 / 4))
    return X, W1, b1, W2, b2, gy, m1.cpu(), m2.cpu(), alpha, talpha


def _op_for_op(X, W1, b1, W2, b2, m1, m2, k, talpha, alpha, depth, A=None):
    if A is None:
        A, _, _ = _graph_dense(m1, m2, k, talpha)
    mp1 = M.MixProp(X.shape[1], W1.shape[0], depth, 0.0, alpha).to(device=X.device, dtype=X.dtype)
    mp2 = M.MixProp(X.shape[1], W1.shape[0], depth, 0.0, alpha).to(device=X.device, dtype=X.dtype)
    for mp, W, b in ((mp1, W1, b1), (mp2, W2, b2)):     # the given tensors themselves, so gradients reach them
        del mp._mlp._mlp.weight, mp._mlp._mlp.bias
        mp._mlp._mlp.weight, mp._mlp._mlp.bias = W, b
    return mp1(X, A) + mp2(X, A.T), (mp1, mp2)


@pytest.mark.parametrize("B,C,n,T,k,depth,dim", [(3, 5, 37, 7, 5, 1, 3), (1, 64, 207, 13, 20, 2, 40), (2, 1, 61, 181, 30, 4, 8),
                                                 (64, 4, 20, 1, 20, 3, 40), (2, 7, 130, 13, 64, 2, 64)])
@pytest.mark.parametrize("want", ["x", "graph", "weights", "x+graph", "x+weights", "graph+weights", "x+graph+weights"])
def test_propagation_and_backward_against_float64(B, C, n, T, k, depth, dim, want):
    X, W1, b1, W2, b2, gy, m1, m2, alpha, talpha = _prop_case(B, C, n, T, k, depth, dim, seed=B * 1000 + n + depth)
    assert bool(_gap_ok(m1, m2, k, talpha).all())
    groups = dict(x=[0], graph=[1, 2], weights=[3, 4, 5, 6])
    leaves = sorted(i for g in want.split("+") for i in groups[g])

    def run_route(dev, dtype, fused):
        ts = [t.to(device=dev, dtype=dtype).clone().requires_grad_(i in leaves)
              for i, t in enumerate((X, m1, m2, W1, b1, W2, b2))]
        x, e1, e2, w1, c1, w2, c2 = ts
        if fused:
            vals, pattern = ops.mtgnn_graph(e1, e2, k, talpha, train=True)
            out = ops.mtgnn_mixprop(x, vals, pattern, k, depth, alpha, w1, c1, w2, c2, train=True)
        else:
            M_req = M._require_cuda
            M._require_cuda = lambda t, name: None
            try:
                out, _ = _op_for_op(x, w1, c1, w2, c2, e1, e2, k, talpha, alpha, depth)
            finally:
                M._require_cuda = M_req
        grads = torch.autograd.grad(out, [ts[i] for i in leaves], gy.to(device=dev, dtype=dtype))
        return out, grads

    of, gf = run_route(DEV, torch.float32, True)
    oo, go = run_route(DEV, torch.float32, False)
    ow, gw = run_route("cpu", D, False)
    _criterion(of, oo, ow, "out")
    for i, (a, b, c) in enumerate(zip(gf, go, gw)):
        _criterion(a, b, c, f"grad {leaves[i]}")


def test_batch_zero_launches_nothing():
    m1, m2 = _embeddings(30, 4, 5)
    vals, pattern = ops.mtgnn_graph(m1, m2, 5, 3.0, train=False)
    x = torch.empty(0, 3, 30, 7, device=DEV)
    W = torch.randn(4, 9, 1, 1, device=DEV)
    b = torch.randn(4, device=DEV)
    with _counted() as cnt:
        y = ops.mtgnn_mixprop(x, vals, pattern, 5, 2, 0.05, W, b, W, b, train=False)
    assert y.shape == (0, 4, 30, 7) and not _ran(cnt)


@pytest.mark.parametrize("kind", ["hub", "full", "empty_rows"])
def test_predefined_graphs(kind):
    """A predefined A (no gradient into it): a hub column every row points at and columns no row chooses, a full A, and A with empty
    rows, through MixProp's algebra against float64."""
    n, B, C, T, depth = 90, 2, 4, 9, 3
    g = torch.Generator().manual_seed(21)
    if kind == "hub":
        A = torch.zeros(n, n)
        A[:, 7] = torch.rand(n, generator=g) + 0.1
        A[torch.arange(n), (torch.arange(n) * 3) % 40] += torch.rand(n, generator=g)
    elif kind == "full":
        A = torch.rand(n, n, generator=g) + 0.01
    else:
        A = (torch.rand(n, n, generator=g) < 0.05).float() * torch.rand(n, n, generator=g)
        A[::3] = 0.0
    X = torch.randn(B, C, n, T, generator=g)
    W1, W2 = 0.3 * torch.randn(5, (depth + 1) * C, 1, 1, generator=g), 0.3 * torch.randn(5, (depth + 1) * C, 1, 1, generator=g)
    b1, b2 = torch.randn(5, generator=g), torch.randn(5, generator=g)
    gy = torch.randn(B, 5, n, T, generator=g)
    pattern, _, vals, w = ops.mtgnn_graph_dense(A.to(DEV))
    if kind == "full":
        assert w == n

    def fused():
        x = X.to(DEV).requires_grad_(True)
        out = ops.mtgnn_mixprop(x, vals, pattern, w, depth, 0.05, *(t.to(DEV) for t in (W1, b1, W2, b2)), train=True)
        return out, torch.autograd.grad(out, x, gy.to(DEV))[0]

    def op(dev, dtype):
        x = X.to(device=dev, dtype=dtype).requires_grad_(True)
        M_req = M._require_cuda
        M._require_cuda = lambda t, name: None
        try:
            out, _ = _op_for_op(x, *(t.to(device=dev, dtype=dtype) for t in (W1, b1, W2, b2)), None, None, 0, 0.0, 0.05, depth,
                                A=A.to(device=dev, dtype=dtype))
        finally:
            M._require_cuda = M_req
        return out, torch.autograd.grad(out, x, gy.to(device=dev, dtype=dtype))[0]

    (of, gf), (oo, go), (ow, gw) = fused(), op(DEV, torch.float32), op("cpu", D)
    _criterion(of, oo, ow, "out")
    _criterion(gf, go, gw, "dX")


# ---- determinism, scaling, launch counts, CUDA graphs -------------------------------------------------------------------------
def _small_model(**kw):
    c = dict(CASES["plain"])
    c["model"] = dict(c["model"], **kw)
    return c, model_for(c, MTGNN, DEV, torch.float32)


def _grads(m):
    """Every parameter's gradient (the layers' _residual_conv is unused with gcn_true, as in the reference: zero)."""
    return {k: p.grad.clone() if p.grad is not None else torch.zeros_like(p) for k, p in m.named_parameters()}


def test_training_forward_equals_no_grad_and_backward_repeats():
    c, m = _small_model()
    X = torch.rand(4, 2, 207, 12, device=DEV)
    m.eval()
    with torch.no_grad():
        want = m(X)
    got = m(X)
    assert torch.equal(got, want)
    grads = []
    for _ in range(2):
        m.zero_grad()
        m(X).square().mean().backward()
        grads.append(_grads(m))
    assert all(torch.equal(grads[0][k], grads[1][k]) for k in grads[0])


@pytest.mark.parametrize("scale", [2.0 ** -24, 2.0 ** 8])
def test_loss_scale_scales_every_gradient_exactly(scale):
    c, m = _small_model()
    X = torch.rand(2, 2, 207, 12, device=DEV)
    Y = torch.randn(2, 10, 207, 1, device=DEV)
    out = {}
    for s in (1.0, scale):
        m.zero_grad()
        ((m(X) - Y).square().sum() * s).backward()
        out[s] = _grads(m)
    for k in out[1.0]:
        assert torch.equal(out[scale][k], out[1.0][k] * scale), k


def test_launch_counts_of_one_forward_and_backward():
    c, m = _small_model()
    X = torch.rand(2, 2, 207, 12, device=DEV)
    L, depth = c["model"]["layers"], c["model"]["gcn_depth"]
    with _counted() as fwd:
        out = m(X)
    assert _ran(fwd) == {**{k: 1 for k in GRAPH}, "k_mtgnn_hop": 2 * depth * L}, _ran(fwd)
    with _counted() as bwd:
        out.sum().backward()
    assert _ran(bwd) == {"k_mtgnn_hop_adjoint": 2 * depth * L, "k_mtgnn_dvals": L, "k_mtgnn_graph_dd": 1, "k_mtgnn_graph_dm": 1}, \
        _ran(bwd)


def test_cuda_graph_replay_of_a_training_step():
    c, m = _small_model()
    X = torch.rand(4, 2, 207, 12, device=DEV)
    Y = torch.randn(4, 10, 207, 1, device=DEV)
    ref = model_for(c, MTGNN, DEV, torch.float32)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)
    opt_ref = torch.optim.Adam(ref.parameters(), lr=1e-3, capturable=True)

    def step(model, o):
        o.zero_grad(set_to_none=False)
        loss = (model(X) - Y).abs().mean()
        loss.backward()
        o.step()
        return loss

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(m, opt)
            step(ref, opt_ref)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step(m, opt)
    for _ in range(3):
        graph.replay()
        want = step(ref, opt_ref)
        torch.cuda.synchronize()
        assert torch.equal(loss, want)
    for (k, p), q in zip(m.named_parameters(), ref.parameters()):
        assert torch.equal(p, q), k


class _Masks:
    """Stands in for mtgnn.py's torch.nn.functional.  "record": every dropout runs as it is and its keep mask is kept, drawn again from
    the same generator state on a tensor of ones (the state rewound, then restored); "replay": every dropout multiplies by the next
    recorded mask and 1 / (1 - p) in the input's dtype."""

    def __init__(self, masks=None):
        self.masks, self.replay, self.i = ([], False, 0) if masks is None else (masks, True, 0)

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)

    def dropout(self, x, p=0.5, training=True, inplace=False):
        if not training or p == 0:
            return torch.nn.functional.dropout(x, p, training)
        if self.replay:
            keep = self.masks[self.i]
            self.i += 1
            return x * keep.to(x.dtype) * (1.0 / (1.0 - p))
        before = torch.cuda.get_rng_state()
        out = torch.nn.functional.dropout(x, p, training)
        after = torch.cuda.get_rng_state()
        torch.cuda.set_rng_state(before)
        keep = torch.nn.functional.dropout(torch.ones_like(x), p, True) != 0
        torch.cuda.set_rng_state(after)
        assert torch.equal(out != 0, keep & (x != 0))             # the mask this call drew
        self.masks.append(keep)
        return out


def test_dropout_masks_replayed_against_float64(monkeypatch):
    """Dropout 0.3 in training: the fused route runs with the masks it draws; the float32 op-for-op route and a float64 op-for-op run
    replay them.  The output and every parameter gradient are held to the criterion."""
    c = dict(CASES["plain"])
    c["model"] = dict(c["model"], dropout=0.3)
    X, Y = (t.to(DEV) for t in inputs(c, 0))

    def step(dtype, fused, masks):
        m = model_for(c, MTGNN, DEV, dtype)
        m.fused_training = fused
        monkeypatch.setattr(M, "F", masks)
        with _counted() as cnt:
            out = m(X.to(dtype))
            (out - Y.to(dtype)).abs().mean().backward()
        monkeypatch.setattr(M, "F", torch.nn.functional)
        grads = {k: p.grad if p.grad is not None else torch.zeros_like(p) for k, p in m.named_parameters()}
        return out.detach(), grads, _ran(cnt)

    rec = _Masks()
    of, gf, ran = step(torch.float32, True, rec)
    assert len(rec.masks) == 1 + c["model"]["layers"] and ran.get("k_mtgnn_dvals") == c["model"]["layers"], ran
    oo, go, ran_o = step(torch.float32, False, _Masks(rec.masks))
    assert not ran_o
    ow, gw, _ = step(D, False, _Masks(rec.masks))
    _criterion(of, oo, ow, "out")
    for k in gw:
        _criterion(gf[k], go[k], gw[k], k)


def test_node_count_mismatch_never_reaches_the_kernels():
    """idx selects 100 of 207 nodes while X keeps all 207: the reference's einsum size error, and no k_mtgnn_* launch."""
    _, m = _small_model()
    X = torch.rand(2, 2, 207, 12, device=DEV)
    with pytest.raises(RuntimeError, match="einsum"), _counted() as cnt:
        m(X, idx=torch.randperm(207, device=DEV)[:100])
    assert not _ran(cnt)


def test_predefined_graph_ignores_node_dim():
    """A predefined A uses no embeddings: node_dim above the graph kernels' 64 still runs fused."""
    c, m = _small_model(build_adj=False, node_dim=80)
    A = (torch.rand(207, 207, device=DEV) < 0.05).float()
    with _counted() as cnt, torch.no_grad():
        m(torch.rand(2, 2, 207, 12, device=DEV), A)
    assert _ran(cnt).get("k_mtgnn_hop") == 2 * c["model"]["gcn_depth"] * c["model"]["layers"], _ran(cnt)


def test_routes_outside_the_envelope():
    c, m = _small_model()
    X = torch.rand(2, 2, 207, 12, device=DEV)
    m.fused_training = False
    with _counted() as cnt:
        m(X).sum().backward()
    assert not _ran(cnt)
    with _counted() as cnt:
        m.double()(X.double()).sum().backward()
    assert not _ran(cnt)
    _, big = _small_model(subgraph_size=65)              # k > 64: op for op
    with _counted() as cnt, torch.no_grad():
        big(X)
    assert not _ran(cnt)
    _, too_many = _small_model(subgraph_size=300)
    with pytest.raises(RuntimeError, match="selected index k out of range"), _counted() as cnt:
        too_many(X)
    assert not _ran(cnt)


def test_abi_errors():
    L_ = _lib.lib()
    assert L_.stmp_mtgnn_supported(207, 20, 40, 32, 2, 64, 19) == _lib.STMP_OK
    for args in ((4097, 20, 40, 32, 2, 1, 1), (207, 65, 40, 32, 2, 1, 1), (207, 20, 65, 32, 2, 1, 1), (207, 20, 40, 65, 2, 1, 1),
                 (207, 20, 40, 32, 5, 1, 1), (207, 20, 40, 32, 0, 1, 1), (10, 11, 4, 4, 1, 1, 1), (207, 20, 40, 32, 2, 1, 0)):
        assert L_.stmp_mtgnn_supported(*args) == _lib.STMP_EUNSUPPORTED, args
    rc = L_.stmp_mtgnn_graph_fwd(10, 3, 4, ctypes.c_float(3.0), None, None, None, None, None, None, None)
    assert rc == _lib.STMP_EINVAL and "NULL" in _lib.last_error()
    rc = L_.stmp_mtgnn_graph_fwd(10, 11, 4, ctypes.c_float(3.0), None, None, None, None, None, None, None)
    assert rc == _lib.STMP_EUNSUPPORTED
    rc = L_.stmp_mtgnn_prop_fwd(1, 65, 10, 4, 3, 2, ctypes.c_float(0.05), None, None, None, None, None)
    assert rc == _lib.STMP_EUNSUPPORTED
