"""The row-split recurrence kernels (gru_rows.cu, lstm_rows.cu, dcrnn_rows.cu, dcrnn_narrow_rows.cu, dcrnn_wide_rows.cu and the host
path behind them) against float64 across their envelopes: outputs and every gradient, at the small and boundary shapes the modules'
routing never reaches, on adversarial graphs.

The modules hand a graph to these kernels only when the one-SM kernels refuse it, so the other row-split tests run at N >= 800.  The C
entries and the autograd Functions take any N, and each kernel cuts the row space its own way: 16-row CTA tiles over N (gru_rows,
lstm_rows) or over the flat B * N rows (dcrnn_rows), 8 consecutive rows of B * N per warp (dcrnn_wide_rows), lane groups of
G = min(32, 2^ceil(log2 B)) windows per row (dcrnn_narrow_rows).  Here they are called below the routing -- `_DcrnnRowsFn`,
`_DcrnnHoistedRowsFn`, `BatchedDCRNN._rows_infer`, `ops.gru_rows_train` / `gru_rows_fwd`, and the LSTM modules (which always take the
row-split kernel) -- where a tile or a warp straddles two windows, the last tile, warp or window group is partial, a graph is smaller
than one warp's rows, and at more than 4 224 rows (2 * 132 tiles of 16), where the grid stride starts.

Numerical criterion (the one of test_gpu_graph_geometry.py): against the float64 oracle (`oracle.recurrent`, run in float64 on the GPU,
autograd for the gradients), the fused path's largest error stays within 4x that of the fp32 op-for-op path (the modules' tiled path
under autograd) plus 2^-20 of the tensor's scale -- for the output, dX, dH / dC where a state is carried, and each parameter's gradient
on its own (the parameter gradients of a narrow model, cout <= 4, share one scale: see `_dcrnn_case`).  Every case also asserts
through the path counters that the row-split kernels it means to test ran, as many times as the launch schedule says, and that no
one-SM kernel did.

The graph family (`make_graph`; `check_family` verifies on the plan's exported forward and transposed CSR that a graph has the
property its kind promises): random, a ring (one entry per row: the gather's 4-unrolled body never runs), rows of every in-degree
residue mod 4 and, separately, of every out-degree residue (the transposed CSR of the backward), an in-hub and an out-hub of N - 1
edges, a last row with nothing but a self loop, duplicate edges with one row longer than N (BatchedDCRNN), a node with in-edges and
no out-edge (the Chebyshev cells).

Largest error ratios of one run on an H100 (80 GB HBM3, 700 W power limit), as printed by `_report` -- observations, not guarantees.
`e / e32` is taken over the comparisons whose error exceeds the 2^-20 floor (below it the ratio says nothing); `used` is the largest
fraction of the allowance 4 e32 + 2^-20 scale that any comparison consumed.  No hub graph needed more than 4x; the narrow kernels at
K = 4 came within 2 % of it and are allowed 8x (see the small-shapes test):
    gru_rows            e / e32 1.18   used 0.28
    lstm_rows           e / e32 1.19   used 0.43
    dcrnn_rows          e / e32 4.26   used 0.52
    dcrnn_narrow_rows   e / e32 5.21   used 0.98   (N = 17, cin 3, cout 2, K 4, B 3, T 5, conv_x_z.weight)
    dcrnn_wide_rows     e / e32 6.39   used 0.65
The whole file ran in 50 s there.
"""
import contextlib
import itertools

import numpy as np
import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, BatchedDCRNN, GConvGRU, GConvLSTM
from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnHoistedRowsFn, _DcrnnRowsFn

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRID_STRIDE_ROWS = 2 * 132 * 16                 # more rows than this and a CTA owns more than one 16-row tile

ONE_SM = ("k_dcrnn_seq", "k_dcrnn_seq_tc", "k_dcrnn_bwd_seq", "k_dcrnn_narrow_seq", "k_dcrnn_narrow_bwd", "k_gru_bwd_seq")
DCRNN_ROWS = ("k_dcrnn_rows_fwd_a", "k_dcrnn_rows_fwd_b", "k_dcrnn_rows_bwd_start", "k_dcrnn_rows_bwd_b", "k_dcrnn_rows_bwd_c",
              "k_dcrnn_rows_bwd_x", "k_dcrnn_nrows_fwd0", "k_dcrnn_nrows_fwd", "k_dcrnn_nrows_seq1", "k_dcrnn_nrows_bwd0",
              "k_dcrnn_nrows_bwd", "k_dcrnn_nrows_bseq1", "k_dcrnn_wrows_image", "k_dcrnn_wrows_fwd0", "k_dcrnn_wrows_fwd",
              "k_dcrnn_wrows_bwd0", "k_dcrnn_wrows_bwd")
CELL_ROWS = ("k_gru_rows_fwd_a", "k_gru_rows_fwd_b", "k_gru_rows_bwd_a", "k_gru_rows_bwd_b", "k_gru_rows_bwd_c", "k_gru_rows_wgrad_reduce",
             "k_lstm_rows_fwd", "k_lstm_rows_bwd_a", "k_lstm_rows_bwd_b", "k_lstm_rows_wgrad_reduce", "k_dcrnn_wgrad")


# ---- helpers: counters, float64, the criterion ----------------------------------------------------------------------------------------
@contextlib.contextmanager
def _counted():
    """Yields a dict that, after the block, holds {kernel: launches during the block}."""
    c0, delta = _lib.path_counters(), {}
    yield delta
    c1 = _lib.path_counters()
    delta.update({k: v - c0.get(k, 0) for k, v in c1.items() if v != c0.get(k, 0)})


def _assert_ran(c, names, want, what):
    """Of the kernels `names`, exactly the launches `want` ran (zero counts dropped), and no one-SM kernel."""
    got = {k: v for k, v in c.items() if k in names}
    assert got == {k: v for k, v in want.items() if v}, (what, got, want)
    assert not [k for k in c if k.split("[")[0] in ONE_SM], (what, c)


@contextlib.contextmanager
def _float64():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)       # the oracle's zeros / scatter buffers
    try:
        yield
    finally:
        torch.set_default_dtype(old)


WORST = {}                                       # family -> [largest e / e32 above the floor, largest used fraction of the allowance, its case]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for fam, (ratio, used, what) in sorted(WORST.items()):
        print(f"\nrows envelope: {fam}: largest e / e32 = {ratio:.2f}, largest used fraction of the allowance = {used:.2f} at {what}")


def _check_err(errs, family, got, ref32, ref64, what, allow=4, scale=None):
    """Appends to `errs` when the fused tensor `got` is further from float64 than `allow` x the fp32 op-for-op path plus 2^-20 of scale
    (the largest magnitude of the float64 tensor unless `scale` is given)."""
    got, ref32, ref64 = got.detach().double(), ref32.detach().double(), ref64.detach()
    assert got.shape == ref64.shape == ref32.shape, (what, got.shape, ref32.shape, ref64.shape)
    if not bool(torch.isfinite(got).all()):
        errs.append((what, "non-finite"))
        return
    e, e32 = float((got - ref64).abs().max()), float((ref32 - ref64).abs().max())
    scale = float(ref64.abs().max()) if scale is None else scale
    floor = 2.0 ** -20 * scale
    w = WORST.setdefault(family, [0.0, 0.0, None])
    if e > floor and e32 > 0:
        w[0] = max(w[0], e / e32)
    if e > w[1] * (4 * e32 + floor):
        w[1:] = [e / (4 * e32 + floor), what]
    if not e <= allow * e32 + floor:
        where = np.unravel_index(int((got - ref64).abs().argmax()), got.shape) if got.dim() else ()
        errs.append((what, "fused / fp32 op-for-op error vs float64", e, e32, scale, "at", tuple(int(i) for i in where)))


def _loss_grads(outs, wgts, leaves):
    sum((o * w).mean() for o, w in zip(outs, wgts)).backward()
    return [None if t is None or t.grad is None else t.grad.detach().clone() for t in leaves]


def _or_zeros(g, like):
    return torch.zeros_like(like) if g is None else g


# ---- 1. the graph family ----------------------------------------------------------------------------------------------------------------
def _unique(src, dst):
    key = src.astype(np.int64) * 1_000_000 + dst
    _, first = np.unique(key, return_index=True)
    keep = np.sort(first)
    return src[keep], dst[keep]


def _distinct(rng, n, k, avoid):
    """k distinct nodes outside `avoid` (fewer when the graph has no more)."""
    free = n - len(set(avoid))
    out = []
    while len(out) < min(k, free):
        for v in rng.integers(0, n, 2 * k + 4).tolist():
            if v not in avoid and v not in out and len(out) < min(k, free):
                out.append(v)
    return np.array(out, dtype=np.int64)


def make_graph(kind, n, seed=0):
    """(src, dst, weight) as numpy arrays.  Every node has in- and out-degree >= 1 (the ring) except `sink`'s node n // 2, which has no
    out-edge; no duplicate edges except in `dups`."""
    rng = np.random.default_rng([seed, n, sum(map(ord, kind))])
    ring = np.arange(n, dtype=np.int64)
    src, dst = ring, (ring + 1) % n
    if kind in ("random", "dups", "sink"):
        src = np.concatenate([src, rng.integers(0, n, 3 * n)])
        dst = np.concatenate([dst, rng.integers(0, n, 3 * n)])
    elif kind == "hubs":                                   # in-hub: N - 1 edges into the last row; out-hub: N - 1 edges out of row 3
        others_in, others_out = np.delete(ring, n - 1), np.delete(ring, 3)
        src = np.concatenate([src, rng.integers(0, n, 2 * n), others_in, np.full(n - 1, 3)])
        dst = np.concatenate([dst, rng.integers(0, n, 2 * n), np.full(n - 1, n - 1), others_out])
    elif kind in ("mod4", "mod4_out"):                     # in- (out-) degree of node i = 1 + i % 9: every residue mod 4, short and long
        a, b = [], []
        for i in range(n):
            other = (i - 1) % n if kind == "mod4" else (i + 1) % n
            cand = _distinct(rng, n, i % 9, (i, other))
            a.append(cand)
            b.append(np.full(cand.size, i, dtype=np.int64))
        extra_src, extra_dst = (a, b) if kind == "mod4" else (b, a)
        src, dst = np.concatenate([src] + extra_src), np.concatenate([dst] + extra_dst)
    elif kind == "lonely":                                 # the last row has nothing but a self loop
        m = n - 1
        r = np.arange(m, dtype=np.int64)
        src = np.concatenate([r, rng.integers(0, m, 3 * m), [m]])
        dst = np.concatenate([(r + 1) % m, rng.integers(0, m, 3 * m), [m]])
    else:
        assert kind == "ring"
    src, dst = _unique(src.astype(np.int64), dst.astype(np.int64))
    if kind == "dups":                                     # every third edge 2..5 times, and n + 5 edges into row 0 from n - 1 sources
        pick = np.arange(0, src.size, 3)
        reps = 1 + pick % 4
        hub = np.arange(n + 5, dtype=np.int64) % (n - 1) + 1
        src = np.concatenate([src, np.repeat(src[pick], reps), hub])
        dst = np.concatenate([dst, np.repeat(dst[pick], reps), np.zeros(n + 5, dtype=np.int64)])
    if kind == "sink":
        keep = src != n // 2
        src, dst = src[keep], dst[keep]
    w = (rng.random(src.size) + 0.1).astype(np.float32)
    return src, dst, w


def _tensors(g):
    src, dst, w = g
    return torch.from_numpy(np.stack([src, dst])).to(DEV), torch.from_numpy(w).to(DEV)


def _row_lengths(plan, op, transposed, off_diagonal):
    rp, col, _, _ = plan.export(op, transposed=transposed)
    rp, col = rp.cpu().numpy().astype(np.int64), col.cpu().numpy().astype(np.int64)
    n = rp.size - 1
    if not off_diagonal:
        return np.diff(rp)
    row = np.repeat(np.arange(n), np.diff(rp))
    return np.bincount(row[row != col], minlength=n)


def check_family(kind, n, g, plan, cheb):
    """The plan's forward and transposed CSR hold the graph as given -- every edge, duplicates included, in both directions -- and the
    graph has what its kind promises.  A DConv plan's operator 0 gathers over in-edges and operator 1 over out-edges; a Chebyshev plan
    drops self loops and adds one diagonal entry per row."""
    src, dst, _ = g
    if cheb:
        keep = src != dst
        src, dst = src[keep], dst[keep]
    indeg, outdeg = np.bincount(dst, minlength=n), np.bincount(src, minlength=n)
    views = [(0, False, indeg), (0, True, outdeg)] + ([] if cheb else [(1, False, outdeg), (1, True, indeg)])
    for op, transposed, deg in views:
        assert np.array_equal(_row_lengths(plan, op, transposed, cheb), deg), (kind, n, "operator", op, "transposed", transposed)
    diag = int(cheb)
    if kind == "ring":
        assert (indeg + diag < 4).all() and (outdeg + diag < 4).all()
    if kind in ("mod4", "dups", "random", "hubs") and n >= 40:
        assert set((indeg + diag) % 4) == {0, 1, 2, 3}
    if kind in ("mod4_out", "dups", "random", "hubs") and n >= 40:
        assert set((outdeg + diag) % 4) == {0, 1, 2, 3}
    if kind == "hubs":
        assert indeg.max() >= n - 1 and outdeg.max() >= n - 1
    if kind == "lonely":
        assert indeg[n - 1] == outdeg[n - 1] == 1 - diag
    if kind == "dups":
        assert indeg.max() > n and src.size > np.unique(src * n + dst).size + n
    if kind == "sink":
        assert outdeg[n // 2] == 0 and indeg[n // 2] >= 1


# ---- 2. BatchedDCRNN on the three row-split kernels, below the routing ----------------------------------------------------------------
def _family(cout):
    return {32: "dcrnn_rows", 64: "dcrnn_wide_rows"}.get(cout, "dcrnn_narrow_rows")


FAMILY_CONFIGS = {                               # (cin, cout, K)
    "dcrnn_rows": [(cin, 32, 2) for cin in (1, 2, 3, 4)],
    "dcrnn_wide_rows": [(cin, 64, K) for K in (2, 3) for cin in (1, 2, 3, 4)],     # (2K-1) cin % 4 != 0 at cin 1, 2, 3: the padded tile
    "dcrnn_narrow_rows": [(1 + (cout + K) % 4, cout, K) for cout in (1, 2, 3, 4) for K in (1, 2, 3, 4)],
}


def _fwd_launches(cout, K, T, chunks=1, nonfinite=False):
    """The forward launch schedule (DESIGN §4k, §4l, §4m).  On a plan with a non-finite value step 0 runs the full chain."""
    steps = T if nonfinite else T - 1
    if cout == 32:
        want = {"k_dcrnn_rows_fwd_a": T, "k_dcrnn_rows_fwd_b": steps}
    elif cout == 64:
        want = {"k_dcrnn_wrows_image": 1, "k_dcrnn_wrows_fwd0": int(not nonfinite), "k_dcrnn_wrows_fwd": 2 * (K - 1) * steps}
    elif K == 1:
        want = {"k_dcrnn_nrows_seq1": 1}
    else:
        want = {"k_dcrnn_nrows_fwd0": int(not nonfinite), "k_dcrnn_nrows_fwd": 2 * (K - 1) * steps}
    return {k: chunks * v for k, v in want.items()}


def _train_launches(cout, K, T):
    """Training forward plus the backward with dX."""
    want = _fwd_launches(cout, K, T)
    if cout == 32:
        want.update({"k_dcrnn_rows_bwd_start": 1, "k_dcrnn_rows_bwd_b": T - 1, "k_dcrnn_rows_bwd_c": T - 1, "k_dcrnn_rows_bwd_x": 1})
    elif cout == 64:
        want.update({"k_dcrnn_wrows_image": 2, "k_dcrnn_wrows_bwd0": 1, "k_dcrnn_wrows_bwd": 2 * (K - 1) * (T - 1)})
    elif K == 1:
        want["k_dcrnn_nrows_bseq1"] = 1
    else:
        want.update({"k_dcrnn_nrows_bwd0": 1, "k_dcrnn_nrows_bwd": 2 * (K - 1) * (T - 1)})
    return want


def _dcrnn_model(cin, cout, K, seed):
    torch.manual_seed(seed)
    m = BatchedDCRNN(cin, cout, K)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith(".bias"):
                p.normal_(0, 0.1)
    return m.to(DEV)


def _dconv_plan(m, g, n, kind):
    ei, ew = _tensors(g)
    plan = m._plan(ei, ew, n)
    check_family(kind, n, g, plan, cheb=False)
    return plan, ei, ew


def _tiled_dcrnn(m, plan, X):
    H, outs = torch.zeros(X.size(0), X.size(2), m.out_channels, device=DEV), []
    for t in range(X.size(1)):
        H = m._tiled_step(plan, X[:, t], H)
        outs.append(H)
    return torch.stack(outs, 1)


def _fused_dcrnn(m, plan, X):
    if m.out_channels == 32:
        return _DcrnnRowsFn.apply(X, *m._params(), plan, m._rows_packed())
    return _DcrnnHoistedRowsFn.apply(X, *m._params(), plan, m.K, m._rows_packed())


def _dcrnn_case(errs, m, plan, ei, ew, n, B, T, seed, what, allow=4):
    """Inference and one training step of the row-split kernels at (B, T, n) against float64: out, dX and every parameter's gradient."""
    cin, cout, K = m.in_channels, m.out_channels, m.K
    fam = _family(cout)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(B, T, n, cin, device=DEV, generator=gen)
    wgt = torch.randn(B, T, n, cout, device=DEV, generator=gen)
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    x64 = X.double().requires_grad_(True)
    with _float64():
        out64 = R.batched_dcrnn(p64, x64, ei, ew.double())
    g64 = _loss_grads([out64], [wgt.double()], [x64] + [p64[k] for k in names])
    x32 = X.clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    out32 = _tiled_dcrnn(m, plan, x32)
    g32 = _loss_grads([out32], [wgt], [x32] + params)
    with torch.no_grad(), _counted() as c:
        inf = m._rows_infer(plan, X)
    _assert_ran(c, DCRNN_ROWS, _fwd_launches(cout, K, T), what)
    xf = X.clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    with _counted() as c:
        out = _fused_dcrnn(m, plan, xf)
        gf = _loss_grads([out], [wgt], [xf] + params)
    _assert_ran(c, DCRNN_ROWS, _train_launches(cout, K, T), what)
    assert c.get("k_spmm", 0) == (0 if cout == 32 else 4 * (K - 1)), (what, c)    # the hoisted X blocks and their adjoint
    assert torch.equal(out.detach(), inf), (what, "training forward differs from inference")
    # A narrow model's parameter gradients are a few numbers each (a bias gradient one to four), every one a sum over all T B N rows
    # that can cancel to a small part of its terms; 2^-20 of such a value is less than any fp32 summation of the rows promises
    # (cout = 1, B = 3: e = 2.4e-9 on a bias gradient that cancelled to 6.0e-4, where the op-for-op path's sum landed within 1.2e-10).
    # They share one scale, the model's largest parameter gradient: the same reduction over the same rows.
    gscale = max(float(t.abs().max()) for t in g64[1:]) if cout <= 4 else None
    for i, (name, got, r32, r64) in enumerate(zip(["out", "dX"] + names, [out] + gf, [out32] + g32, [out64] + g64)):
        _check_err(errs, fam, got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (name,), allow, gscale if i >= 2 else None)
    return X, inf


SMALL_N = (1, 2, 7, 8, 9, 15, 16, 17, 31, 33, 207)


@pytest.mark.parametrize("n", SMALL_N)
@pytest.mark.parametrize("family", list(FAMILY_CONFIGS))
def test_dcrnn_small_and_boundary_shapes_vs_float64(family, n):
    """Tiles and 8-row warps that straddle windows (N % 16, N % 8 != 0), partial last tiles and warps, graphs smaller than one warp's
    rows, T = 1 (no recurrent launch) and T = 2 (exactly one).  The configurations cycle so that every (cin, cout, K) of a family meets
    several (N, B, T)."""
    g = make_graph("random", n)
    cfgs = FAMILY_CONFIGS[family]
    errs, plans = [], {}
    for j, (B, T) in enumerate(itertools.product((1, 2, 3), (1, 2, 5))):
        cin, cout, K = cfgs[(j + 9 * SMALL_N.index(n)) % len(cfgs)]
        m = _dcrnn_model(cin, cout, K, seed=n + j)
        if "plan" not in plans:
            plans["plan"] = _dconv_plan(m, g, n, "random")
        plan, ei, ew = plans["plan"]
        # K = 4: the third-order blocks 2 P (2 P P U - U) - U cancel, and the hand-written adjoint associates them differently from
        # autograd.  In one run conv_x_z.weight at N = 17, (cin, cout, K) = (3, 2, 4), B = 3, T = 5 used 0.98 of the 4x allowance, and
        # the family's largest error was 5.2x the op-for-op path's, so K = 4 is allowed 8x.
        _dcrnn_case(errs, m, plan, ei, ew, n, B, T, 100 * n + j, (family, n, cin, cout, K, B, T), allow=8 if K == 4 else 4)
    assert not errs, errs[:6]


WINDOW_COUNTS = (1, 2, 3, 5, 6, 7, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65)


@pytest.mark.parametrize("B", WINDOW_COUNTS)
@pytest.mark.parametrize("cout", [1, 3])
def test_narrow_window_group_edges_vs_float64(cout, B):
    """dcrnn_narrow_rows.cu: lane groups of G = min(32, 2^ceil(log2 B)) windows, ceil(B / G) window groups per row.  Every B whose last
    lane group or window group is partial, B = 32 exactly and 63 / 65; cout = 3 is the one padded width (CP = 4).  A window's result
    does not depend on the windows beside it: "every multiply-add of a (window, row) happens in CSR entry order whatever B is"."""
    n, K, T, cin = 40, 3, 3, 2
    g = make_graph("mod4", n)
    m = _dcrnn_model(cin, cout, K, seed=cout)
    plan, ei, ew = _dconv_plan(m, g, n, "mod4")
    errs = []
    X, inf = _dcrnn_case(errs, m, plan, ei, ew, n, B, T, 7 * B + cout, ("narrow window groups", cout, B))
    assert not errs, errs[:6]
    for b in sorted({0, B // 2, B - 1, min(B - 1, 31), min(B - 1, 32)}):
        with torch.no_grad(), _counted() as c:
            alone = m._rows_infer(plan, X[b:b + 1])
        _assert_ran(c, DCRNN_ROWS, _fwd_launches(cout, K, T), (cout, B, b))
        assert torch.equal(alone[0], inf[b]), ("window", b, "of", B, "differs from the same window run alone")


DCRNN_KINDS = ("random", "ring", "mod4", "mod4_out", "hubs", "lonely", "dups")
KIND_CONFIG = {"dcrnn_rows": (3, 32, 2), "dcrnn_wide_rows": (3, 64, 3), "dcrnn_narrow_rows": (2, 3, 3)}
N_STRIDED = 4300                                 # more than GRID_STRIDE_ROWS rows already at B = 1


@pytest.mark.parametrize("n", [129, N_STRIDED])
@pytest.mark.parametrize("kind", DCRNN_KINDS)
@pytest.mark.parametrize("family", list(FAMILY_CONFIGS))
def test_dcrnn_graph_kinds_vs_float64(family, kind, n):
    assert N_STRIDED > GRID_STRIDE_ROWS
    cin, cout, K = KIND_CONFIG[family]
    g = make_graph(kind, n)
    m = _dcrnn_model(cin, cout, K, seed=n)
    plan, ei, ew = _dconv_plan(m, g, n, kind)
    errs = []
    _dcrnn_case(errs, m, plan, ei, ew, n, 2, 3, n + len(kind), (family, kind, n))
    assert not errs, errs[:6]


@pytest.mark.parametrize("family", list(FAMILY_CONFIGS))
def test_dcrnn_zero_in_degree_node_inside_a_tile_gives_the_reference_non_finite_pattern(family):
    """Node 21 of 40 has no in-edge, so DConv's 1 / deg_in is inf on its out-edges; it sits in the middle of a 16-row tile and of an
    8-row warp group, and with B = 3 the tiles straddle windows.  The non-finite values spread one hop per basis from there, as in the
    reference; the rest stay finite and are held to the criterion."""
    n, B, T, bad = 40, 3, 2, 21
    cin, cout, _ = KIND_CONFIG[family]
    K = 2
    ring = np.arange(n, dtype=np.int64)
    src, dst = np.concatenate([ring, ring]), np.concatenate([(ring + 1) % n, (ring + 7) % n])
    keep = dst != bad
    ei = torch.from_numpy(np.stack([src[keep], dst[keep]])).to(DEV)
    ew = torch.ones(ei.size(1), device=DEV)
    m = _dcrnn_model(cin, cout, K, seed=5)
    plan = m._plan(ei, ew, n)
    X = torch.randn(B, T, n, cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    with torch.no_grad():
        ref32 = R.batched_dcrnn(sd, X, ei, ew)
        with _float64():
            ref64 = R.batched_dcrnn({k: v.double() for k, v in sd.items()}, X.double(), ei, ew.double())
    fin = torch.isfinite(ref32)
    assert torch.equal(fin, torch.isfinite(ref64)) and bool(fin.any()) and not bool(fin.all())
    errs = []
    for train in (False, True):
        with torch.set_grad_enabled(train), _counted() as c:
            got = (_fused_dcrnn(m, plan, X) if train else m._rows_infer(plan, X)).detach()
        _assert_ran(c, DCRNN_ROWS, _fwd_launches(cout, K, T, nonfinite=True), (family, train))
        assert torch.equal(torch.isfinite(got), fin), (family, train, "non-finite pattern differs from the reference's")
        _check_err(errs, _family(cout), got[fin], ref32[fin], ref64[fin], (family, "finite values", train))
    assert not errs, errs


@pytest.mark.parametrize("cout,K", [(2, 3), (3, 4), (64, 2), (64, 3)])
def test_hoisted_inference_chunks_with_a_short_last_chunk_are_bit_identical(monkeypatch, cout, K):
    """`ops.dcrnn_hoisted_rows_fwd` cuts the windows of a no_grad call so that the hoisted X blocks stay under `_NROWS_XBUF_BYTES`.
    B = 7 as chunks of 3, 3 and 1 (the last one reuses the front of the buffer and a scratch sized for 3) equals the unchunked call bit
    for bit, for materialised windows and for windows indexed in a resident series."""
    n, B, T, cin = 77, 7, 4, 3
    g = make_graph("mod4", n)
    m = _dcrnn_model(cin, cout, K, seed=K)
    plan, ei, ew = _dconv_plan(m, g, n, "mod4")
    series = torch.randn(40, n, cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    starts = torch.tensor([3, 30, 0, 17, 36, 8, 21], device=DEV)
    X = torch.stack([series[i:i + T] for i in starts.tolist()])
    with torch.no_grad():
        with _counted() as c:
            whole = m._rows_infer(plan, X)
        _assert_ran(c, DCRNN_ROWS, _fwd_launches(cout, K, T), (cout, K, "unchunked"))
        assert torch.equal(m._rows_infer(plan, series, win_start=starts, horizon=T), whole)
        monkeypatch.setattr(ops, "_NROWS_XBUF_BYTES", 3 * T * n * (2 * K - 1) * cin * 4)
        with _counted() as c:
            cut = m._rows_infer(plan, X)
        _assert_ran(c, DCRNN_ROWS, _fwd_launches(cout, K, T, chunks=3), (cout, K, "chunked"))
        assert c.get("k_spmm") == 3 * 2 * (K - 1)
        assert torch.equal(cut, whole)
        with _counted() as c:
            cut = m._rows_infer(plan, series, win_start=starts, horizon=T)
        _assert_ran(c, DCRNN_ROWS, _fwd_launches(cout, K, T, chunks=3), (cout, K, "chunked, indexed"))
        assert torch.equal(cut, whole)


# ---- 3. GConvGRU, GConvLSTM and GCLSTM on gru_rows.cu / lstm_rows.cu --------------------------------------------------------------------
CELLS = {"gconv_gru": GConvGRU, "gconv_lstm": GConvLSTM, "gc_lstm": GCLSTM}
ORACLE = {"gconv_gru": R.gconv_gru_cell, "gconv_lstm": R.gconv_lstm_cell, "gc_lstm": R.gc_lstm_cell}
CELL_FAMILY = {"gconv_gru": "gru_rows", "gconv_lstm": "lstm_rows", "gc_lstm": "lstm_rows"}


def _cell_model(name, cin, K, norm, bias, seed):
    torch.manual_seed(seed)
    m = CELLS[name](cin, 32, K, normalization=norm, bias=bias).to(DEV)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("bias") or k.startswith("b_"):
                p.copy_(torch.randn_like(p) * 0.1)
    return m


def _lam(norm):
    return torch.tensor(1.7, device=DEV) if norm == "rw" else None


def _cell_step(name, m, X, ei, ew, state, lam, fused, train=True):
    """One cell step -> list of outputs ([H'] or [H', C']).  `fused`: the row-split kernels -- the GRU's through `ops`, below the
    module's routing (which prefers the one-SM kernel on small graphs); the LSTM modules take the row-split kernel on any graph.
    Otherwise the module's op-for-op path under autograd."""
    m.fused_training = fused
    if name == "gconv_gru" and fused:
        plan = m._cheb_plan(ei, ew, X.size(0), m.normalization, lam)
        w, b = m._rows_packed()
        if not train:
            return [ops.gru_rows_fwd(plan, m.K - 1, X, state[0], w, b)]
        spec, params = m._param_spec(rows=True)
        return [ops.gru_rows_train(plan, m.K - 1, X, state[0], w, b, spec, params)]
    out = m(X, ei, ew, *state, lambda_max=lam)
    return [out] if name == "gconv_gru" else list(out)


def _cell_launches(name, K, state, wants, train=True):
    """The row-split launches of one step (DESIGN §4i, §4j); `wants` = (dX, dH[, dC]) wanted."""
    if name == "gconv_gru":
        want = {"k_gru_rows_fwd_a": 1, "k_gru_rows_fwd_b": int(state[0] is not None)}
        if train:
            want.update({"k_gru_rows_bwd_a": 1, "k_gru_rows_bwd_b": int(state[0] is not None),
                         "k_gru_rows_bwd_c": int(K == 2 and (wants[0] or wants[1])), "k_dcrnn_wgrad": 1, "k_gru_rows_wgrad_reduce": 1})
        return want
    want = {"k_lstm_rows_fwd": 1}
    if train:
        gather = K == 2 and (wants[1] or (wants[0] and name == "gconv_lstm"))
        want.update({"k_lstm_rows_bwd_a": 1, "k_lstm_rows_bwd_b": int(gather), "k_dcrnn_wgrad": 1, "k_lstm_rows_wgrad_reduce": 1})
    return want


def _oracle_step(name, p64, x, ei, ew, state, norm, lam):
    zeros = torch.zeros(x.size(0), 32, dtype=torch.float64, device=DEV)
    st = [zeros if s is None else s for s in state]
    out = ORACLE[name](p64, x, ei, ew.double(), *st, lambda_max=None if lam is None else lam.double(), normalization=norm)
    return [out] if name == "gconv_gru" else list(out)


def _cell_case(errs, name, m, ei, ew, n, norm, given, wants, seed, what, allow=4):
    """One step of a cell on the row-split kernels against float64.  `given`: which of (H[, C]) are passed (else None); `wants`: which of
    (X, H[, C]) require a gradient.  Unwanted gradients must come back as None, wanted ones are held to the criterion."""
    cin, K, ns = m.in_channels, m.K, len(given)
    lam = _lam(norm)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(n, cin, device=DEV, generator=gen)
    S = [0.5 * torch.randn(n, 32, device=DEV, generator=gen) for _ in range(ns)]
    wgts = [torch.randn(n, 32, device=DEV, generator=gen) for _ in range(ns)]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    wants = [wants[0]] + [w and gv for w, gv in zip(wants[1:], given)]

    def leaves(dtype, need):
        x = X.to(dtype, copy=True).requires_grad_(need[0])
        st = [S[i].to(dtype, copy=True).requires_grad_(need[1 + i]) if given[i] else None for i in range(ns)]
        return x, st
    everything = [True] * (1 + ns)
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    x64, s64 = leaves(torch.float64, everything)
    with _float64():
        o64 = _oracle_step(name, p64, x64, ei, ew, s64, norm, lam)
    g64 = _loss_grads(o64, [w.double() for w in wgts], [x64] + s64 + [p64[k] for k in names])
    x32, s32 = leaves(torch.float32, everything)
    m.zero_grad(set_to_none=True)
    o32 = _cell_step(name, m, x32, ei, ew, s32, lam, fused=False)
    g32 = _loss_grads(o32, wgts, [x32] + s32 + params)
    with torch.no_grad(), _counted() as c:
        inf = _cell_step(name, m, X, ei, ew, [S[i] if given[i] else None for i in range(ns)], lam, fused=True, train=False)
    _assert_ran(c, CELL_ROWS, _cell_launches(name, K, s32, wants, train=False), what)
    xf, sf = leaves(torch.float32, wants)
    m.zero_grad(set_to_none=True)
    with _counted() as c:
        of = _cell_step(name, m, xf, ei, ew, sf, lam, fused=True)
        gf = _loss_grads(of, wgts, [xf] + sf + params)
    _assert_ran(c, CELL_ROWS, _cell_launches(name, K, sf, wants), what)
    assert "k_spmm" not in c, (what, c)
    fam = CELL_FAMILY[name]
    for i, (a, b) in enumerate(zip(of, inf)):
        assert torch.equal(a.detach(), b), (what, "training forward differs from inference", i)
    for i, (a, r32, r64) in enumerate(zip(of, o32, o64)):
        _check_err(errs, fam, a, r32, r64, what + (("H'", "C'")[i],), allow)
    for label, want, got, r32, r64 in zip(["dX", "dH", "dC"][:1 + ns] + names, wants + [True] * len(names), gf, g32, g64):
        if not want:
            assert got is None, (what, label, "unwanted gradient")
            continue
        assert got is not None, (what, label)
        _check_err(errs, fam, got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (label,), allow)


CELL_KINDS = ("ring", "mod4", "mod4_out", "hubs", "lonely", "sink")
CELL_GEOMETRIES = ([("ring", n) for n in (1, 15, 16, 17, 33)] + [("mod4", 17), ("mod4", 33)] + [(k, 129) for k in CELL_KINDS]
                   + [("mod4_out", N_STRIDED), ("hubs", N_STRIDED)])
CELL_CONFIGS = list(itertools.product((1, 4, 5, 15, 16), (1, 2)))      # (cin, K); K = 2 at cin = 16 fills the 96-column weight row


@pytest.mark.parametrize("kind,n", CELL_GEOMETRIES, ids=[f"{k}-N{n}" for k, n in CELL_GEOMETRIES])
@pytest.mark.parametrize("name", list(CELLS))
def test_cells_vs_float64(name, kind, n):
    """Every (cin, K) on every geometry; the normalization, the bias and which states are given cycle so that each meets each."""
    g = make_graph(kind, n)
    ei, ew = _tensors(g)
    gi = CELL_GEOMETRIES.index((kind, n))
    ns = 1 if name == "gconv_gru" else 2
    errs, checked = [], False
    for idx, (cin, K) in enumerate(CELL_CONFIGS):
        norm = ("sym", "rw", None)[(idx + gi) % 3]
        if n == 1 and norm is None:              # L = D - A of a single node is 0, and lambda_max = 2 max(L) = 0 divides it
            norm = "sym"
        bias = bool((idx + gi // 3) % 2)
        given = [bool((idx + gi) >> i & 1) for i in range(ns)]
        m = _cell_model(name, cin, K, norm, bias, seed=idx + n)
        if not checked:
            check_family(kind, n, g, m._cheb_plan(ei, ew, n, norm, _lam(norm)), cheb=True)
            checked = True
        _cell_case(errs, name, m, ei, ew, n, norm, given, [True] * (1 + ns), 31 * n + idx, (name, kind, n, cin, K, norm, bias, tuple(given)))
    assert not errs, errs[:6]


@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("name", list(CELLS))
def test_cell_state_and_gradient_flags_vs_float64(name, K):
    """Every combination the kernels specialise on: H (and C) None or given, and the gradients of X, H, C wanted or not."""
    n, cin, kind = 33, 5, "mod4"
    g = make_graph(kind, n)
    ei, ew = _tensors(g)
    ns = 1 if name == "gconv_gru" else 2
    m = _cell_model(name, cin, K, "sym", True, seed=K)
    check_family(kind, n, g, m._cheb_plan(ei, ew, n, "sym", None), cheb=True)
    errs, seen = [], set()
    for given in itertools.product((False, True), repeat=ns):
        for wants in itertools.product((False, True), repeat=1 + ns):
            eff = (given, (wants[0],) + tuple(w and gv for w, gv in zip(wants[1:], given)))
            if eff in seen:
                continue
            seen.add(eff)
            _cell_case(errs, name, m, ei, ew, n, "sym", list(given), list(wants), len(seen), (name, K, given, wants))
    assert not errs, errs[:6]


@pytest.mark.parametrize("name", list(CELLS))
def test_cell_carried_recurrence_vs_float64(name):
    """Five steps with H (and C) fed back and one backward through all of them: the state gradient that enters a cell's backward is
    the one the next cell produced."""
    n, cin, K, steps, kind = 129, 4, 2, 5, "mod4_out"
    g = make_graph(kind, n)
    ei, ew = _tensors(g)
    ns = 1 if name == "gconv_gru" else 2
    m = _cell_model(name, cin, K, "sym", True, seed=11)
    check_family(kind, n, g, m._cheb_plan(ei, ew, n, "sym", None), cheb=True)
    gen = torch.Generator(device=DEV).manual_seed(2)
    X = torch.randn(steps, n, cin, device=DEV, generator=gen)
    S0 = [0.5 * torch.randn(n, 32, device=DEV, generator=gen) for _ in range(ns)]
    wgts = [torch.randn(n, 32, device=DEV, generator=gen) for _ in range(steps * ns)]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]

    def run(dtype, step):
        x = X.to(dtype, copy=True).requires_grad_(True)
        s0 = [s.to(dtype, copy=True).requires_grad_(True) for s in S0]
        state, outs = s0, []
        for t in range(steps):
            state = step(x[t], state)
            outs += state
        return x, s0, outs
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    with _float64():
        x64, s64, o64 = run(torch.float64, lambda x, st: _oracle_step(name, p64, x, ei, ew, st, "sym", None))
    g64 = _loss_grads(o64, [w.double() for w in wgts], [x64] + s64 + [p64[k] for k in names])
    m.zero_grad(set_to_none=True)
    x32, s32, o32 = run(torch.float32, lambda x, st: _cell_step(name, m, x, ei, ew, st, None, fused=False))
    g32 = _loss_grads(o32, wgts, [x32] + s32 + params)
    m.zero_grad(set_to_none=True)
    with _counted() as c:
        xf, sf, of = run(torch.float32, lambda x, st: _cell_step(name, m, x, ei, ew, st, None, fused=True))
        gf = _loss_grads(of, wgts, [xf] + sf + params)
    _assert_ran(c, CELL_ROWS, {k: steps * v for k, v in _cell_launches(name, K, sf, [True] * (1 + ns)).items()}, name)
    errs, fam = [], CELL_FAMILY[name]
    for label, got, r32, r64 in zip(["out"] + ["dX", "dH0", "dC0"][:1 + ns] + names, [torch.stack(of)] + gf,
                                    [torch.stack(o32)] + g32, [torch.stack(o64)] + g64):
        _check_err(errs, fam, got, _or_zeros(r32, got), _or_zeros(r64, got.double()), (name, "recurrence", label))
    assert not errs, errs[:6]
