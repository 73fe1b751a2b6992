"""The SpMM + wgmma Chebyshev LSTM routes and the pointwise gate kernels against float64 across their envelopes, the routes every
GConvLSTM / GCLSTM / GConvGRU call outside the row-split and one-SM kernels takes:

- `_LstmCellFn` (GConvLSTM training at out_channels 32 / 64 with K (in + out) a multiple of 64 up to 512): the basis built in place by
  `stmp_spmm`, `stmp_gemm_lstm_f32`, and the hand-written backward -- the recomputed GEMM, `stmp_lstm_gate_bwd`, the two prescaled
  dS halves and the transposed in-place Chebyshev adjoint.  Outputs, dX, dH, dC and every parameter gradient.
- `stmp_gemm_lstm_f32` for `no_grad` GConvLSTM and GCLSTM: K (in + out) on and off the 64-wide k-block, rows on each side of the
  128-row tile, and the 2048-node rule at 64 channels (`ops.lstm_rows_for_no_grad`).
- `stmp_lstm_ifc` / `stmp_lstm_oh` / `stmp_gru_zr` / `stmp_gru_out`, the `no_grad` fallback at any other width: peephole channel
  indices other than 16, odd element counts, and more elements than one pass of their capped grid (132 * 32 blocks of 256).
- A state shared across a batch -- X (B, N, F) with H, C (N, out), which the reference broadcasts -- on every route, dH / dC included.
- The `ops` guards that refuse operands a kernel would overrun, before any launch.

Criterion (the one of test_gpu_rows_envelope.py): against the float64 oracle (`oracle.recurrent`, float64 on the GPU, autograd for
gradients) the route's largest error stays within 4x that of the fp32 op-for-op path (the same module with `fused_training = False`
under autograd) plus 2^-20 of the tensor's scale.  Every case asserts through the path counters the exact launches of the route it
claims, and that no row-split or one-SM kernel ran.

Tensors computed through the fp16 hi/lo split GEMMs -- H' and C' of `stmp_gemm_lstm_f32`, and every gradient of `_LstmCellFn`, which
flows from the recomputed pre-activations and the two dS halves -- are allowed SPLIT_ALLOW = 4 C_SPLIT / 1.5 ~ 21x instead of 4x.  That
is the criterion's 4x times the ratio of the two per-element bounds of test_gpu_split_precision.py (`_bound`): the split GEMM's error is
at most C_SPLIT 2^-22 (|A||W|)_mn, fp32's own accumulation at most 1.5 2^-22 (|A||W|)_mn for the same operands.  The first run
measured 5.8x on the inference GEMM's outputs and 19.6x on a weight gradient of `_LstmCellFn`.

Largest error ratios of one run on an H100 (80 GB HBM3, 700 W power limit), as printed by `_report` -- observations, not guarantees.
`used` is, as in the rows envelope, the largest fraction of the 4x allowance 4 e32 + 2^-20 scale that any comparison consumed; above 1
it is within SPLIT_ALLOW:
    lstm_cell_fn     e / e32 19.60   used 2.80   (64, 64, K 4, 43 nodes, B = 1, conv_x_c.lins.3.weight)
    gemm_lstm        e / e32  5.81   used 1.19   (GConvLSTM (64, 32, K 5), 2 x 43 rows, H')
    lstm_pointwise   e / e32  1.00   used 0.23
    gru_pointwise    e / e32  0.00   used 0.19   (every error below the 2^-20 floor)
The whole file ran in 18 s there.
"""
import itertools

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvGRU, GConvLSTM
from test_gpu_split_precision import C_SPLIT
from test_gpu_rows_envelope import WORST, _check_err, _counted, _float64, _loss_grads, _or_zeros, _tensors, check_family, make_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"
POINTWISE_GRID = 132 * 32 * 256                  # elements one pass of the pointwise kernels' grid covers; beyond it the grid stride runs
PATH = ("k_spmm", "k_gemm_split", "k_lstm_gate_bwd", "k_lstm_ifc", "k_lstm_oh", "k_gru_zr", "k_gru_out")
FUSED_CELLS = ("k_lstm_rows", "k_lstm_wide_rows", "k_gru_rows", "k_gru_wide_rows", "k_gru_seq", "k_gru_bwd", "k_dcrnn", "k_tgcn")
MODULES = {"gconv_lstm": GConvLSTM, "gc_lstm": GCLSTM, "gconv_gru": GConvGRU}
ORACLE = {"gconv_lstm": R.gconv_lstm_cell, "gc_lstm": R.gc_lstm_cell, "gconv_gru": R.gconv_gru_cell}
FAMILIES = ("lstm_cell_fn", "gemm_lstm", "lstm_pointwise", "gru_pointwise")
SPLIT_ALLOW = 4 * C_SPLIT / 1.5
ALLOW = {"lstm_cell_fn": SPLIT_ALLOW, "gemm_lstm": SPLIT_ALLOW, "lstm_pointwise": 4, "gru_pointwise": 4}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for fam in FAMILIES:
        if fam in WORST:
            ratio, used, what = WORST[fam]
            print(f"\ncheb lstm envelope: {fam}: largest e / e32 = {ratio:.2f}, largest used fraction of the allowance = {used:.2f} at {what}")


def _assert_path(c, want, what):
    """Of the route's kernels exactly the launches `want` ran, and no row-split or one-SM cell kernel."""
    got = {k: v for k, v in c.items() if k in PATH}
    assert got == {k: v for k, v in want.items() if v}, (what, got, want)
    assert not [k for k in c if k.startswith(FUSED_CELLS)], (what, c)


_GRAPHS = {}


def _graph(kind, n):
    if (kind, n) not in _GRAPHS:
        _GRAPHS[(kind, n)] = make_graph(kind, n)
    return _GRAPHS[(kind, n)]


def _model(name, cin, cout, K, norm, bias, seed):
    torch.manual_seed(seed)
    m = MODULES[name](cin, cout, K, normalization=norm, bias=bias).to(DEV)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("bias") or k.startswith("b_"):
                p.copy_(torch.randn_like(p) * 0.1)
    return m


def _lam(norm):
    return torch.tensor(1.7, device=DEV) if norm == "rw" else None


def _setup(name, cin, cout, K, norm, bias, kind, n, seed):
    g = _graph(kind, n)
    ei, ew = _tensors(g)
    m = _model(name, cin, cout, K, norm, bias, seed)
    check_family(kind, n, g, m._cheb_plan(ei, ew, n, norm, _lam(norm)), cheb=True)
    return m, ei, ew


def _nstates(name):
    return 1 if name == "gconv_gru" else 2


def _inputs(name, cout, lead, n, cin, given, shared, steps, seed):
    """X (steps, *lead, n, cin) and the initial states: None where not given, (n, cout) when shared across the batch."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(steps, *lead, n, cin, device=DEV, generator=gen)
    slead = () if shared else tuple(lead)
    S = [0.5 * torch.randn(*slead, n, cout, device=DEV, generator=gen) if gv else None for gv in given]
    wgts = [torch.randn(*lead, n, cout, device=DEV, generator=gen) for _ in range(steps * _nstates(name))]
    return X, S, wgts


def _run(step, X, S0, need, dtype):
    """Steps of a cell with the state carried; -> (leaves [x, given states..], outputs of every step)."""
    x = X.to(dtype, copy=True).requires_grad_(need[0])
    s0 = [None if s is None else s.to(dtype, copy=True).requires_grad_(w) for s, w in zip(S0, need[1:])]
    state, outs = s0, []
    for t in range(X.size(0)):
        state = step(x[t], state)
        outs += state
    return [x] + [s for s in s0 if s is not None], outs


def _module_step(name, m, ei, ew, lam):
    def step(x, st):
        out = m(x, ei, ew, *st, lambda_max=lam)
        return [out] if name == "gconv_gru" else list(out)
    return step


def _oracle_step(name, p64, ei, ew, norm, lam, n, cout):
    def step(x, st):
        st = [torch.zeros(n, cout, dtype=torch.float64, device=DEV) if s is None else s for s in st]
        out = ORACLE[name](p64, x, ei, ew.double(), *st, lambda_max=None if lam is None else lam.double(), normalization=norm)
        return [out] if name == "gconv_gru" else list(out)
    return step


def _case(errs, fam, name, m, ei, ew, X, S, wgts, norm, train, want_path, what, wants=None):
    """The route (`fused_training = True`, under autograd when `train`, else `no_grad`) against float64 and the fp32 op-for-op path:
    every step's outputs and, when training, the gradient of each wanted input and of every parameter."""
    n, cout = X.size(-2), m.out_channels
    lam = _lam(norm)
    given = [s is not None for s in S]
    wants = [True] * (1 + len(S)) if wants is None else wants
    need = [wants[0]] + [w and gv for w, gv in zip(wants[1:], given)]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    with _float64():
        l64, o64 = _run(_oracle_step(name, p64, ei, ew, norm, lam, n, cout), X, S, [True] * (1 + len(S)), torch.float64)
    g64 = _loss_grads(o64, [w.double() for w in wgts], l64 + [p64[k] for k in names]) if train else None
    m.fused_training = False
    m.zero_grad(set_to_none=True)
    l32, o32 = _run(_module_step(name, m, ei, ew, lam), X, S, [True] * (1 + len(S)), torch.float32)
    g32 = _loss_grads(o32, wgts, l32 + params) if train else None
    m.fused_training = True
    m.zero_grad(set_to_none=True)
    with torch.set_grad_enabled(train), _counted() as c:
        lf, of = _run(_module_step(name, m, ei, ew, lam), X, S, need if train else [False] * len(need), torch.float32)
        gf = _loss_grads(of, wgts, lf + params) if train else None
    _assert_path(c, want_path, what)
    for i, (a, r32, r64) in enumerate(zip(of, o32, o64)):
        assert a.shape == r64.shape, (what, "output", i, a.shape, r64.shape)
        _check_err(errs, fam, a, r32, r64, what + (f"out{i}",), ALLOW[fam])
    if not train:
        return
    labels = ["dX"] + [lab for lab, gv in zip(["dH", "dC"], given) if gv]
    wanted = [need[0]] + [w for w, gv in zip(need[1:], given) if gv]
    for label, want, got, r32, r64 in zip(labels + names, wanted + [True] * len(names), gf, g32, g64):
        if not want:
            assert got is None, (what, label, "unwanted gradient")
            continue
        assert got is not None and got.shape == r64.shape, (what, label)
        _check_err(errs, fam, got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (label,), ALLOW[fam])


# ---- 1. _LstmCellFn: GConvLSTM training on the basis buffer, the fused GEMM and the hand-written backward -----------------------------
def _cell_fn_launches(K, steps=1):
    return {"k_spmm": 2 * (K - 1) * steps, "k_gemm_split": 4 * steps, "k_lstm_gate_bwd": steps}


CELL_FN_CONFIGS = [(32, 32, K) for K in range(1, 9)] + [(16, 32, 4), (32, 64, 2), (32, 64, 4)] + [(64, 64, K) for K in range(1, 5)]
STATE_MODES = ("none", "given", "grad")          # H / C None, given, given with requires_grad
LAYOUTS = ("2d", "3d", "shared", "3d1")           # (N, F); (3, N, F) with (3, N, out) states; (3, N, F) with (N, out) states; (1, N, F)


def _layout(layout):
    return {"2d": ((), False), "3d": ((3,), False), "shared": ((3,), True), "3d1": ((1,), False)}[layout]


@pytest.mark.parametrize("cin,cout,K", CELL_FN_CONFIGS, ids=[f"{a}-{b}-K{c}" for a, b, c in CELL_FN_CONFIGS])
def test_lstm_cell_fn_vs_float64(cin, cout, K):
    """Every configuration inside the route's gates, K (in + out) = 512 included (dS halves of 256 columns).  The normalization, the
    bias, the state mode and the layout cycle so that each meets each; K = 1 has no propagation at all."""
    i = CELL_FN_CONFIGS.index((cin, cout, K))
    errs = []
    for j in range(2):
        norm = ("sym", "rw", None)[(i + j) % 3]
        bias = bool((i + j) % 2)
        mode = STATE_MODES[(i + 2 * j) % 3]
        layout = LAYOUTS[(i + j) % 4]
        lead, shared = _layout(layout)
        n = (129, 43, 127)[(i + j) % 3] if not lead else 43
        m, ei, ew = _setup("gconv_lstm", cin, cout, K, norm, bias, "mod4" if n < 100 else "hubs", n, seed=i * 7 + j)
        X, S, wgts = _inputs("gconv_lstm", cout, lead, n, cin, [mode != "none"] * 2, shared, 1, 10 * i + j)
        wants = [True, mode == "grad", mode == "grad"]
        _case(errs, "lstm_cell_fn", "gconv_lstm", m, ei, ew, X, S, wgts, norm, True, _cell_fn_launches(K),
              ("cell_fn", cin, cout, K, norm, bias, mode, layout, n), wants)
    assert not errs, errs[:6]


ROW_COUNTS = [(1, 1), (1, 127), (1, 128), (1, 129), (3, 43), (1, 1009), (4, 1024), (4, 8192)]   # (B, N): B N = 1 .. 32 768


@pytest.mark.parametrize("B,n", ROW_COUNTS, ids=[f"B{b}-N{n}" for b, n in ROW_COUNTS])
def test_lstm_cell_fn_row_counts_vs_float64(B, n):
    """B N rows on each side of the GEMM's 128-row tile, and the weight gradient's chunking (`_chunked_tn`): one chunk (a prime row
    count), 16 chunks (4 096 rows) and 128 (32 768)."""
    K = 3
    kind = "ring" if n == 1 else ("random" if n > 1000 else "mod4")
    m, ei, ew = _setup("gconv_lstm", 32, 32, K, "sym", True, kind, n, seed=n)
    lead = () if B == 1 and n % 2 else (B,)
    X, S, wgts = _inputs("gconv_lstm", 32, lead, n, 32, [True, True], B > 1 and n % 2 == 1, 1, n + B)
    errs = []
    _case(errs, "lstm_cell_fn", "gconv_lstm", m, ei, ew, X, S, wgts, "sym", True, _cell_fn_launches(K), ("cell_fn rows", B, n))
    assert not errs, errs[:6]


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("cin,cout,K", [(32, 32, 4), (32, 64, 2)])
def test_lstm_cell_fn_carried_sequence_vs_float64(cin, cout, K, shared):
    """Three steps with H and C fed back, one backward through all of them (the state gradients that enter a step's backward come from
    the next step); from a state shared across a batch of 3 when `shared`."""
    n = 129
    m, ei, ew = _setup("gconv_lstm", cin, cout, K, "sym", True, "sink", n, seed=K)
    X, S, wgts = _inputs("gconv_lstm", cout, (3,) if shared else (), n, cin, [True, True], shared, 3, K + shared)
    errs = []
    _case(errs, "lstm_cell_fn", "gconv_lstm", m, ei, ew, X, S, wgts, "sym", True, _cell_fn_launches(K, 3), ("cell_fn carried", cin, cout, K, shared))
    assert not errs, errs[:6]


@pytest.mark.parametrize("cin,cout,K", [(32, 32, 9), (4, 32, 3), (16, 16, 4)])
def test_lstm_cell_fn_neighbours_take_autograd(cin, cout, K):
    """Just outside the gates -- K (in + out) = 576 > 512, K (in + out) = 108 not a multiple of 64, out_channels 16 -- training runs the
    op-for-op autograd path: no fused GEMM, no gate backward, the same bits as `fused_training = False`."""
    n = 43
    m, ei, ew = _setup("gconv_lstm", cin, cout, K, "sym", True, "mod4", n, seed=1)
    X, S, wgts = _inputs("gconv_lstm", cout, (), n, cin, [True, True], False, 1, 3)
    outs = []
    for fused in (True, False):
        m.fused_training = fused
        m.zero_grad(set_to_none=True)
        with _counted() as c:
            leaves, o = _run(_module_step("gconv_lstm", m, ei, ew, None), X, S, [True] * 3, torch.float32)
            g = _loss_grads(o, wgts, leaves + list(m.parameters()))
        assert not [k for k in c if k in ("k_gemm_split", "k_lstm_gate_bwd", "k_lstm_ifc", "k_lstm_oh")], (cin, cout, K, c)
        assert c.get("k_spmm") == 2 * (K - 1), c
        outs.append([t.detach() for t in o] + g)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ---- 2. stmp_gemm_lstm_f32: no_grad GConvLSTM and GCLSTM --------------------------------------------------------------------------------
def _gemm_launches(K):
    return {"k_spmm": K - 1, "k_gemm_split": 1}


GEMM_N = (127, 128, 129, 257, 43)


@pytest.mark.parametrize("cout", [32, 64])
@pytest.mark.parametrize("name", ["gconv_lstm", "gc_lstm"])
def test_gemm_lstm_inference_vs_float64(name, cout):
    """K = 1 .. 5 and in_channels 4 / 8 / 20 / 32 / 64: K (in + out) on and off the 64-wide k-block (e.g. (4, 32, 3) -> 108), 2-D X where
    the row-split cell refuses it (K >= 3 or in_channels > 16), 3-D X (where it must), and states shared across the batch."""
    errs = []
    for idx, (K, cin) in enumerate(itertools.product(range(1, 6), (4, 8, 20, 32, 64))):
        norm = ("sym", "rw", None)[idx % 3]
        bias = bool(idx % 2)
        two_d = (K >= 3 or cin > 16) and idx % 3 != 0
        lead, shared = ((), False) if two_d else ((2,), bool(idx % 2))
        n = GEMM_N[idx % len(GEMM_N)]
        given = [bool(idx % 4), bool(idx % 4 != 1)]
        m, ei, ew = _setup(name, cin, cout, K, norm, bias, "mod4" if n < 200 else "hubs", n, seed=idx)
        X, S, wgts = _inputs(name, cout, lead, n, cin, given, shared, 1, idx)
        _case(errs, "gemm_lstm", name, m, ei, ew, X, S, wgts, norm, False, _gemm_launches(K), (name, cin, cout, K, norm, bias, lead, shared, n))
    assert not errs, errs[:6]


@pytest.mark.parametrize("n", [ops.LSTM_WIDE_ROWS_GEMM_NODES - 1, ops.LSTM_WIDE_ROWS_GEMM_NODES])
@pytest.mark.parametrize("name", ["gconv_lstm", "gc_lstm"])
def test_gemm_lstm_wide_rows_rule(name, n):
    """At 64 channels, K <= 2, in_channels 8, 2-D X: the row-split cell below 2048 nodes, the SpMM + wgmma route from 2048 on (16 full
    row tiles); both against float64."""
    m, ei, ew = _setup(name, 8, 64, 2, "sym", True, "random", n, seed=n)
    X, S, wgts = _inputs(name, 64, (), n, 8, [True, True], False, 1, n)
    errs = []
    if n >= ops.LSTM_WIDE_ROWS_GEMM_NODES:
        _case(errs, "gemm_lstm", name, m, ei, ew, X, S, wgts, "sym", False, _gemm_launches(2), (name, "wide rule", n))
    else:
        with torch.no_grad(), _counted() as c:
            m(X[0], ei, ew, *S)
        assert c.get("k_lstm_wide_rows_fwd") == 1 and "k_gemm_split" not in c, c
    assert not errs, errs[:6]


# ---- 3. the pointwise gate kernels: no_grad at any other width ---------------------------------------------------------------------
def _pointwise_launches(name, K):
    if name == "gconv_gru":
        return {"k_spmm": 2 * (K - 1), "k_gru_zr": 1, "k_gru_out": 1}
    return {"k_spmm": K - 1, "k_lstm_ifc": 1, "k_lstm_oh": 1}


POINTWISE_CONFIGS = {                             # (cin, cout, K, layout)
    "gconv_lstm": [(4, co, K, lay) for co, K, lay in ((1, 2, "2d"), (3, 3, "3d"), (16, 1, "shared"), (33, 2, "2d"), (48, 4, "shared"),
                                                      (100, 3, "2d"), (128, 2, "3d"))] + [(5, 32, 3, "2d"), (18, 32, 2, "shared")],
    "gc_lstm": [(3, co, K, lay) for co, K, lay in ((1, 3, "2d"), (3, 2, "shared"), (16, 4, "3d"), (33, 1, "2d"), (48, 2, "2d"),
                                                   (100, 3, "shared"), (128, 2, "2d"))] + [(5, 32, 3, "2d"), (18, 32, 2, "shared")],
    "gconv_gru": [(4, 16, 3, "2d"), (3, 33, 4, "shared"), (5, 32, 3, "2d"), (2, 64, 1, "3d"), (1, 100, 2, "2d"), (6, 1, 3, "shared"),
                  (4, 48, 2, "3d")],
}


@pytest.mark.parametrize("name", list(POINTWISE_CONFIGS))
def test_pointwise_gates_vs_float64(name):
    """Peephole channel indices i % out_channels for widths 1 .. 128, in_channels % 4 != 0 at 32 channels (no fused GEMM), odd element
    counts (127 or 43 rows times an odd width), 3-D X and shared states; GConvGRU at K >= 3, widths other than 32 / 64, and 3-D X."""
    fam = "gru_pointwise" if name == "gconv_gru" else "lstm_pointwise"
    errs = []
    for idx, (cin, cout, K, layout) in enumerate(POINTWISE_CONFIGS[name]):
        norm = ("sym", "rw", None)[idx % 3]
        lead, shared = _layout(layout)
        n = 127 if not lead else 43
        given = [bool(idx % 3)] * _nstates(name)
        m, ei, ew = _setup(name, cin, cout, K, norm, bool(idx % 2), "mod4_out" if n < 100 else "hubs", n, seed=idx)
        X, S, wgts = _inputs(name, cout, lead, n, cin, given, shared, 1, idx)
        _case(errs, fam, name, m, ei, ew, X, S, wgts, norm, False, _pointwise_launches(name, K), (name, cin, cout, K, norm, layout, n))
    assert not errs, errs[:6]


@pytest.mark.parametrize("name", list(POINTWISE_CONFIGS))
def test_pointwise_gates_grid_stride_vs_float64(name):
    """50 000 nodes x 33 channels = 1 650 000 elements, more than one pass of the capped grid: the grid-stride loop's second pass, with
    a state shared across a batch of 2 for the LSTM cells."""
    n, cout, K = 50_000, 33, 2
    assert n * cout > POINTWISE_GRID
    m, ei, ew = _setup(name, 3, cout, K, "sym", True, "random", n, seed=5)
    lead, shared = ((), False) if name == "gconv_gru" else ((2,), True)
    X, S, wgts = _inputs(name, cout, lead, n, 3, [True] * _nstates(name), shared, 1, 5)
    errs = []
    fam = "gru_pointwise" if name == "gconv_gru" else "lstm_pointwise"
    _case(errs, fam, name, m, ei, ew, X, S, wgts, "sym", False, _pointwise_launches(name, K), (name, "grid stride", n))
    assert not errs, errs[:6]


# ---- 4. the ops guards: refused before any launch -----------------------------------------------------------------------------------------
def test_ops_guards_refuse_a_state_of_too_few_rows_before_any_launch():
    rows, Co, K = 96, 32, 64
    z = lambda *s: torch.zeros(*s, device=DEV)
    g, st, v = z(rows, Co), z(rows // 3, Co), z(1, Co)
    packed = ops.gemm_prepack(z(K, 4 * Co))
    bad = [lambda: ops.gemm_lstm(z(rows, K), packed, K, Co, None, st, *[v] * 7),
           lambda: ops.gemm_lstm(z(rows, K), packed, K, Co, z(Co), g, *[v] * 7),
           lambda: ops.lstm_ifc(g, g, g, st, *[v] * 5), lambda: ops.lstm_ifc(g, g, g, g, v, v, v, v, z(2 * Co)),
           lambda: ops.lstm_oh(g, st, v, v), lambda: ops.gru_zr(g, g, st), lambda: ops.gru_out(g, g, st), lambda: ops.gru_out(g, st, g),
           lambda: ops.lstm_gate_bwd(z(rows, 4 * Co), g, g, st, None, *[v] * 7),
           lambda: ops.lstm_gate_bwd(z(rows // 3, 4 * Co), g, g, None, None, *[v] * 7)]
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    for i, call in enumerate(bad):
        with pytest.raises(RuntimeError, match="elements, the kernel indexes"):
            call()
    assert _lib.launch_count() == n0
    with _counted() as c:                                           # and the same calls with matching operands launch
        ops.gemm_lstm(z(rows, K), packed, K, Co, None, g, *[v] * 7)
        ops.lstm_ifc(g, g, g, g, *[v] * 5)
        ops.gru_out(g, g, g)
    assert c == {"k_gemm_split": 1, "k_lstm_ifc": 1, "k_gru_out": 1}, c
