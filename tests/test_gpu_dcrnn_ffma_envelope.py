"""The FFMA DCRNN kernel (dcrnn_seq.cu: `k_dcrnn_seq<OUT, RT, NW>`) and the two backwards `_DcrnnSeqFn` pairs with it against float64
across their envelope.  This is the wide-state route that is neither wgmma, narrow nor row-split: `DCRNN` / `BatchedDCRNN` take it
whenever `dcrnn_seq_supported` holds but the wgmma kernel does not -- 16 or 32 hidden channels at K != 2 (the reference's example
model `DCRNN(4, 32, 1)`), 32 channels at K = 2 on 208-256 nodes or on a graph of <= 207 nodes too dense for the 8-bit graph images,
16 channels up to 512 nodes.  In training its stash feeds the persistent backward `k_dcrnn_bwd_seq` (K = 2, 32 channels, while
`fits_one_sm` holds: up to 232 nodes at cin 1-2, 216 at cin 3-4), on a CTA pair or one CTA, reading the transposed graph staged in
shared memory or from the global CSR; otherwise the per-step loop of `_DcrnnSeqFn.backward` (`gru_bwd_carry`, the transposed SpMMs of
`_x_blocks_adjoint`, `gru_bwd_zr`, `_weight_grads`).

A Python mirror of the launch logic -- `shape_ok`, `make_layout` and `launch_rt` (dcrnn_seq.cu), the TMA condition of
`stmp_dcrnn_seq_fwd`, `dcrnn_tc_supported` through the graph-image mirror of test_gpu_graph_geometry.py, `fits_one_sm`,
`graph_in_smem` and the CTA-pair rule of `seq_impl` (dcrnn_bwd.cu) -- predicts for every call the forward instance (OUT, RT, NW), TMA
or plain X loads, the largest window length T the double-buffered X fits, and for training calls the backward route.  Each case
asserts that `dcrnn_seq_supported`, `dcrnn_bwd_supported` and the path counters (`k_dcrnn_seq[<OUT,RT,NW>]`, `k_dcrnn_seq[x-plain]`,
`k_dcrnn_bwd_seq[cluster2]`, `[graph-global]`, `k_gru_bwd_carry`, `k_gru_bwd_zr`, `k_spmm`) agree with it.  `_report` checks at the
end of the module that all 10 instances, both X-load modes, the four persistent-backward routes, the per-step backward and the tiled
route past the X buffer launched.

Numerical criterion (the one of test_gpu_rows_envelope.py, whose helpers this file imports): against the float64 oracle
(`oracle.recurrent`, run in float64 on the GPU, autograd for the gradients), the fused path's largest error stays within 4x that of
the fp32 op-for-op path (the module's tiled path under autograd) plus 2^-20 of the tensor's scale -- for the output, dX, dH0 and each
parameter gradient on its own scale, under a randomly weighted loss.  No case needs more.

Largest error ratios of one run on an H100 (80 GB HBM3, 700 W power limit), as printed by `_report` -- observations, not guarantees.
`e / e32` is taken over the comparisons whose error exceeds the 2^-20 floor; `used` is the largest fraction of the allowance
4 e32 + 2^-20 scale that any comparison consumed:
    forward                     e / e32 2.01   used 0.38   (N = 1, cin 4, cout 32, K = 3, out)
    persistent backward         e / e32 2.01   used 0.41   (207 nodes, a 509-entry row, cin 3, conv_x_r.bias)
    per-step backward           e / e32 6.73   used 0.77   (N = 90, cin 2, cout 16, K = 4, dH0)
    tiled route (T past limit)  e / e32 0.00   used 0.18
    example model (chickenpox)  e / e32 0.00   used 0.11
The whole file (60 cases) ran in 18 s there.
"""
import functools

import numpy as np
import pytest
import torch

from gconvgru_seq import chickenpox_train_split
from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN, BatchedDCRNN
from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnSeqFn
from test_gpu_dcrnn_narrow_envelope import _bwd_launches, _edges, _oracle_seq, _tiled
from test_gpu_graph_geometry import E_DENSE as E_IMAGE, _option, bwd_staged, image_fits, make_graph as geo_graph, ncol_of
from test_gpu_rows_envelope import (WORST, _check_err, _counted, _dcrnn_model, _float64, _loss_grads, _or_zeros, _tensors, check_family,
                                    make_graph)

pytestmark = pytest.mark.gpu
DEV = "cuda"
FAM = "ffma: "                                   # prefix of this file's families in WORST


# ---- the mirror of the launch logic ------------------------------------------------------------------------------------------------
SMEM = 232448                                    # kMaxSmem: the 227 KB opt-in limit per CTA
BWD_SMEM = 227 * 1024 - 16                       # kBwdSmemMax
BWD_THREADS = 512                                # kBwdThreads
ROW_MAPS = ((1, 8), (2, 8), (4, 8), (7, 8), (4, 16))   # launch_rt's (RT, NW) in order; rows covered = NW * (128 / OUT) * RT
IMG_ROW_MAX = 508                                # the graph image's 7-bit group count: at most 127 groups of four entries per row
SUPPORT_T = 12                                   # the window length stmp_dcrnn_seq_supported checks the layout at


@functools.lru_cache(maxsize=None)
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _align(v, a):
    return (v + a - 1) // a * a


def shape_ok(n, cin, cout, K):
    return cout in (16, 32) and 1 <= cin <= 4 and 1 <= K <= 4 and n <= 16 * (128 // cout) * 4


def layout_bytes(n, nnz, cin, cout, K, T):
    """make_layout: S [N][LD], the weights [LD][3 cout], the biases, the task starts and order, both operators' entries with at most
    3 pad entries per task, then two X buffers of T N cin floats and the two mbarriers."""
    CP = _align(cout + cin, 4)
    LD = (2 * K - 1) * CP
    off = (_align(n * LD * 4, 128) + _align(LD * 3 * cout * 4, 128) + _align(3 * cout * 4, 128) + _align((2 * n + 1) * 4, 16)
           + _align(2 * n * 4, 16) + _align((nnz[0] + nnz[1] + 6 * n + 4) * 8, 16))
    return _align(off, 128) + 2 * _align(T * n * cin * 4, 128) + 16


def max_T(n, nnz, cin, cout, K):
    """The largest T for which layout_bytes fits (-1: not even T = 0)."""
    rest = SMEM - layout_bytes(n, nnz, cin, cout, K, 0)
    return -1 if rest < 0 else (rest // 2) // 128 * 128 // (4 * n * cin)


def instance(n, cout):
    """launch_rt: the first (RT, NW) whose rows cover N."""
    for rt, nw in ROW_MAPS:
        if n <= nw * (128 // cout) * rt:
            return (cout, rt, nw)
    return None


def fits_one_sm(n, cin):
    ncol, rg = ncol_of(cin), (n + 7) // 8
    base = 4 * (3 * 32 * ncol + rg * 8 * ncol + 2 * 32 * (rg * 8 + 4) + n * 36)
    return rg * (ncol // 8) <= BWD_THREADS and base <= BWD_SMEM and 8 * n * (cin + 32) <= 100 * 1024


def _nnz(plan, transposed):
    return tuple(int(plan.export(op, transposed=transposed)[0][-1]) for op in (0, 1))


def _longest_row(plan):
    return max(int(np.diff(plan.export(op)[0].cpu().numpy()).max()) for op in (0, 1))


def plain_loads(n, cin, T, x, indexed):
    """The negation of stmp_dcrnn_seq_fwd's TMA condition: whole 16-byte windows at a 16-byte aligned start."""
    tma = (T * n * cin) % 4 == 0 and x.data_ptr() % 16 == 0 and (not indexed or (n * cin) % 4 == 0)
    return not tma


class Expect:
    """The mirror's prediction for one call on `plan`, after checking the library's support answers against it."""

    def __init__(self, plan, cin, cout, K, B, T, tc=True, fused_bwd=True, bwd_split=True):
        n = plan.num_nodes
        self.n, self.cin, self.cout, self.K, self.B, self.T = n, cin, cout, K, B, T
        nf, nb = _nnz(plan, False), _nnz(plan, True)
        ok = shape_ok(n, cin, cout, K)
        has_image = K == 2 and cout == 32 and image_fits(n, 2, sum(nf)) and _longest_row(plan) <= IMG_ROW_MAX
        assert ops.gru_seq_supported(plan, 2, cin, 32) == (ok and has_image and cin <= 4) or not (K == 2 and cout == 32)
        self.tc = ok and tc and has_image
        self.tmax = max_T(n, nf, cin, cout, K) if ok else -1
        supported = ok and (self.tc or self.tmax >= SUPPORT_T)
        with _option("dcrnn_tc", int(tc), 1):
            assert ops.dcrnn_seq_supported(plan, cin, cout, K) == supported, (n, nf, cin, cout, K, self.tmax)
        bwd_ok = K == 2 and cout == 32 and 1 <= cin <= 4 and fits_one_sm(n, cin)
        assert ops.dcrnn_bwd_supported(plan, cin, cout, K) == bwd_ok, (n, cin, cout, K)
        self.fwd = None if self.tc or not ok or T > self.tmax else instance(n, cout)
        self.persistent = fused_bwd and bwd_ok
        self.split = self.persistent and bwd_split and 2 * B <= _sms() and n >= 16
        self.staged = self.persistent and bwd_staged(n, cin, list(nb))

    def bwd_route(self):
        if not self.persistent:
            return ("bwd", "per-step")
        return ("bwd", "pair" if self.split else "one", "staged" if self.staged else "global")

    def label(self):
        f = "fwd<%d,%d,%d>" % self.fwd if self.fwd else ("fwd wgmma" if self.tc else "fwd refused")
        return f"{f} Tmax {self.tmax} " + "/".join(self.bwd_route()[1:])


LAUNCHED = set()
REACHABLE = ({("fwd", co, rt, nw) for co in (16, 32) for rt, nw in ROW_MAPS} | {("x", "tma"), ("x", "plain")}
             | {("bwd", s, g) for s in ("pair", "one") for g in ("staged", "global")} | {("bwd", "per-step"), ("tiled",)})


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    failed_before = request.session.testsfailed
    yield
    for fam, (ratio, used, what) in sorted(WORST.items()):
        if fam.startswith(FAM):
            print(f"\nffma envelope: {fam[len(FAM):]}: largest e / e32 = {ratio:.2f}, largest used fraction of the allowance = {used:.2f} "
                  f"at {what}")
    print(f"\nffma envelope: launched: {sorted(LAUNCHED, key=str)}")
    # checked when every test of this module was selected and none of them failed (a failing case stops before its later launches)
    here = {it.originalname for it in request.session.items if it.module is request.module}
    every = {k for k, v in vars(request.module).items() if k.startswith("test_") and callable(v)}
    failed_here = request.session.testsfailed - failed_before
    print(f"ffma envelope: launch check {'runs' if here == every and not failed_here else 'skipped'} "
          f"({len(here)} of {len(every)} tests selected, {failed_here} failed here)")
    if here == every and not failed_here:
        assert LAUNCHED == REACHABLE, ("never launched", sorted(REACHABLE - LAUNCHED, key=str))


def _assert_fwd(c, e, plain, what):
    """One k_dcrnn_seq at the mirror's instance, plain X loads exactly when predicted, no wgmma kernel, no SpMM."""
    assert e.fwd is not None, (what, "the mirror refuses the forward")
    got = {k: v for k, v in c.items() if k.startswith("k_dcrnn_seq")}
    want = {"k_dcrnn_seq": 1, "k_dcrnn_seq[<%d,%d,%d>]" % e.fwd: 1}
    if plain:
        want["k_dcrnn_seq[x-plain]"] = 1
    assert got == want, (what, got, want)
    assert "k_spmm" not in c and not [k for k in c if k.startswith(("k_dcrnn_narrow", "k_dcrnn_rows", "k_dcrnn_nrows", "k_dcrnn_wrows"))], \
        (what, c)
    LAUNCHED.update({("fwd",) + e.fwd, ("x", "plain" if plain else "tma")})


def _assert_bwd(c, e, what):
    """The backward of `_DcrnnSeqFn`: k_dcrnn_bwd_seq with the predicted pair / graph counters, or the per-step branch with
    `_bwd_launches`' counts -- never both, and no forward kernel."""
    got = {k: v for k, v in c.items() if k.startswith(("k_dcrnn_bwd_seq", "k_gru_bwd_carry", "k_gru_bwd_zr", "k_spmm"))}
    if e.persistent:
        want = {"k_dcrnn_bwd_seq": 1}
        if e.split:
            want["k_dcrnn_bwd_seq[cluster2]"] = 1
        if not e.staged:
            want["k_dcrnn_bwd_seq[graph-global]"] = 1
    else:
        want = _bwd_launches(None, e.K, e.T)
    assert got == want, (what, got, want)
    assert not [k for k in c if k.startswith(("k_dcrnn_seq", "k_dcrnn_narrow"))], (what, c)
    LAUNCHED.add(e.bwd_route())


# ---- one case: inference and a training step against float64 ------------------------------------------------------------------------
def _case(errs, m, plan, ei, ew, B, T, seed, what, h0=False, want_dx=True, train=True, tc=False, fused_bwd=True, route=None):
    """`ops.dcrnn_seq_fwd` and `_DcrnnSeqFn` at (B, T) on `plan` (the wgmma kernel switched off unless `tc`): the launches the mirror
    predicts, the training forward equal to inference bit for bit, out, dX, dH0 and every parameter gradient against float64, and where
    the persistent backward runs on a CTA pair, the same step on one CTA per window bit for bit.  `route`: the backward route the case
    was built to reach, checked against the mirror.  Returns (X, H0, inference)."""
    cin, cout, K = m.in_channels, m.out_channels, m.K
    e = Expect(plan, cin, cout, K, B, T, tc=tc, fused_bwd=fused_bwd)
    assert route is None or e.bwd_route() == route, (what, route, e.bwd_route())
    what = what + (e.label(),)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(B, T, plan.num_nodes, cin, device=DEV, generator=gen)
    wgt = torch.randn(B, T, plan.num_nodes, cout, device=DEV, generator=gen)
    H0 = 0.5 * torch.randn(B, plan.num_nodes, cout, device=DEV, generator=gen) if h0 else None
    plain = plain_loads(plan.num_nodes, cin, T, X, False)
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    with torch.no_grad(), _option("dcrnn_tc", int(tc), 1), _counted() as c:
        inf = ops.dcrnn_seq_fwd(plan, X, *m._params(), K, h0=H0)
    _assert_fwd(c, e, plain, what)
    p64 = {k: v.detach().double().requires_grad_(train) for k, v in m.state_dict().items()}
    x64 = X.double().requires_grad_(train)
    h64 = None if H0 is None else H0.double().requires_grad_(train)
    with _float64(), torch.set_grad_enabled(train):
        out64 = _oracle_seq(p64, x64, ei, ew.double(), h64)
    if not train:
        with torch.no_grad():
            out32 = _tiled(m, plan, X, H0)
        _check_err(errs, FAM + "forward", inf, out32, out64.detach(), what + ("out",))
        return X, H0, inf
    g64 = _loss_grads([out64], [wgt.double()], [x64, h64] + [p64[k] for k in names])
    x32 = X.clone().requires_grad_(True)
    h32 = None if H0 is None else H0.clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    out32 = _tiled(m, plan, x32, h32)
    g32 = _loss_grads([out32], [wgt], [x32, h32] + params)
    runs = []
    for split in ((1, 0) if e.split else (1,)):
        es = e if split else Expect(plan, cin, cout, K, B, T, tc=tc, fused_bwd=fused_bwd, bwd_split=False)
        xf = X.clone().requires_grad_(want_dx)
        hf = None if H0 is None else H0.clone().requires_grad_(True)
        m.zero_grad(set_to_none=True)
        old, _DcrnnSeqFn.fused_backward = _DcrnnSeqFn.fused_backward, fused_bwd
        try:
            with _option("dcrnn_tc", int(tc), 1), _option("dcrnn_bwd_split", split, 1):
                with _counted() as cf:
                    out = _DcrnnSeqFn.apply(xf, hf, *m._params(), plan, K, m._weight_image())
                with _counted() as cb:
                    gf = _loss_grads([out], [wgt], [xf, hf] + params)
        finally:
            _DcrnnSeqFn.fused_backward = old
        _assert_fwd(cf, e, plain, what)
        _assert_bwd(cb, es, what + (es.label(),))
        assert torch.equal(out.detach(), inf), (what, "training forward differs from inference")
        if not want_dx:
            assert gf[0] is None, (what, "dX computed though X does not require grad")
        runs.append([out.detach()] + gf)
    for a, b in zip(*runs) if len(runs) == 2 else ():
        assert (a is None and b is None) or torch.equal(a, b), (what, "CTA pair differs from one CTA")
    bfam = FAM + ("persistent backward" if e.persistent else "per-step backward")
    _check_err(errs, FAM + "forward", runs[0][0], out32, out64, what + ("out",))
    for i, (label, got, r32, r64) in enumerate(zip(["dX", "dH0"] + names, runs[0][1:], g32, g64)):
        if (i == 0 and not want_dx) or (i == 1 and H0 is None):
            continue
        _check_err(errs, bfam, got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (label,))
    return X, H0, inf


def _plan_of(m, g, n, kind=None):
    ei, ew = _tensors(g)
    plan = m._plan(ei, ew, n)
    if kind is not None:
        check_family(kind, n, g, plan, cheb=False)
    return plan, ei, ew


def _long_row(n, length):
    """The ring plus duplicate edges into row 0 until it holds `length` entries (BatchedDCRNN semantics): a sparse graph without a
    graph image (more than 508 entries in one row)."""
    ring = np.arange(n, dtype=np.int64)
    hub = np.arange(length - 1, dtype=np.int64) % (n - 1) + 1
    src, dst = np.concatenate([ring, hub]), np.concatenate([(ring + 1) % n, np.zeros(length - 1, np.int64)])
    return src, dst, (np.random.default_rng([n, length]).random(src.size) + 0.1).astype(np.float32)


# ---- 1. the mirror itself ----------------------------------------------------------------------------------------------------------
def test_mirror_limits():
    """The limits quoted in DESIGN §5, from the restatement alone: the X buffer's T at 228 nodes, cin 2, K 2 and 4N edges per
    operator; the persistent backward's 232 / 216-node limits; the instance thresholds; max_T against a search."""
    assert max_T(228, (912, 912), 2, 32, 2) == 17
    for cin, last in ((1, 232), (2, 232), (3, 216), (4, 216)):
        assert fits_one_sm(last, cin) and not fits_one_sm(last + 1, cin), cin
    assert [instance(n, 32)[1:] for n in (32, 33, 64, 65, 128, 129, 224, 225, 256)] == \
        [(1, 8), (2, 8), (2, 8), (4, 8), (4, 8), (7, 8), (7, 8), (4, 16), (4, 16)]
    assert [instance(n, 16)[1:] for n in (64, 65, 128, 129, 256, 257, 448, 449, 512)] == \
        [(1, 8), (2, 8), (2, 8), (4, 8), (4, 8), (7, 8), (7, 8), (4, 16), (4, 16)]
    assert instance(257, 32) is None and instance(513, 16) is None
    for n, nnz, cin, cout, K in ((1, (1, 1), 1, 16, 1), (228, (912, 912), 2, 32, 2), (61, (300, 300), 3, 16, 4), (500, (2000, 2000), 1, 16, 2)):
        t = max_T(n, nnz, cin, cout, K)
        assert layout_bytes(n, nnz, cin, cout, K, t) <= SMEM < layout_bytes(n, nnz, cin, cout, K, t + 1)


# ---- 2. forward: the (cout, K, cin) grid on both sides of every row-mapping threshold ---------------------------------------------
GRID_N = {32: (1, 2, 32, 33, 64, 65, 128, 129, 224, 225, 256), 16: (1, 2, 64, 65, 128, 129, 256, 257, 448, 449, 512)}
GRID = [(cout, K) for cout in (16, 32) for K in (1, 2, 3, 4)]


@pytest.mark.parametrize("cout,K", GRID, ids=[f"cout{co}-K{K}" for co, K in GRID])
def test_forward_grid_vs_float64(cout, K):
    """Every N of GRID_N at this (cout, K), with cin cycling through 1..4 so that every cin meets small and large graphs; a shape
    whose layout does not fit is refused by `dcrnn_seq_fwd` as the mirror says.  K = 2 at 32 channels runs with the wgmma kernel
    switched off where it would take the graph."""
    errs, ran = [], set()
    for i, n in enumerate(GRID_N[cout]):
        cin = 1 + (i + K) % 4
        m = _dcrnn_model(cin, cout, K, seed=n + 10 * K + cout)
        plan, ei, ew = _plan_of(m, make_graph("random", n, seed=K), n, "random" if n >= 40 else None)
        B, T = 2, 3
        e = Expect(plan, cin, cout, K, B, T, tc=False)
        if e.fwd is None:
            with _option("dcrnn_tc", 0, 1), pytest.raises(_lib.StmpUnsupported):
                ops.dcrnn_seq_fwd(plan, torch.zeros(B, T, n, cin, device=DEV), *m._params(), K)
            continue
        _case(errs, m, plan, ei, ew, B, T, n + cin, ("grid", n, cin, cout, K), h0=bool(i % 2), train=False)
        ran.add(cin)
    assert ran == {1, 2, 3, 4}, ran
    assert not errs, errs[:6]


# ---- 3. the graph family, and the densest graph the layout holds ------------------------------------------------------------------
KINDS = ("hubs", "mod4", "mod4_out", "lonely", "dups", "ring")
KIND_SHAPES = [(129, 2, 32, 3), (449, 1, 16, 2), (225, 3, 32, 2)]      # (N, cin, cout, K): RT 7 / 8 warps, RT 4 / 16 warps, both


@pytest.mark.parametrize("kind", KINDS)
def test_graph_kinds_vs_float64(kind):
    """Inference and a training step (the per-step backward; at 225 nodes and cin 3 past the persistent backward's 216) on each graph
    kind of test_gpu_rows_envelope.py."""
    errs = []
    for j, (n, cin, cout, K) in enumerate(KIND_SHAPES):
        m = _dcrnn_model(cin, cout, K, seed=n + j)
        plan, ei, ew = _plan_of(m, make_graph(kind, n, seed=j), n, kind)
        _case(errs, m, plan, ei, ew, 2, 3, n + len(kind), ("kind", kind, n, cin, cout, K), h0=j == 1, route=("bwd", "per-step"))
    assert not errs, errs[:6]


def _max_edges(n, cin, cout, K, T):
    """The largest E (one entry per edge in each operator) whose layout fits at window length T."""
    E = (SMEM - layout_bytes(n, (0, 0), cin, cout, K, T)) // 16
    while layout_bytes(n, (E + 1, E + 1), cin, cout, K, T) <= SMEM:
        E += 1
    while layout_bytes(n, (E, E), cin, cout, K, T) > SMEM:
        E -= 1
    return E


DENSE = [(64, 2, 16, 4, ("bwd", "per-step")), (160, 1, 32, 3, ("bwd", "per-step")), (225, 2, 32, 2, ("bwd", "pair", "global"))]


@pytest.mark.parametrize("case", DENSE, ids=[f"N{c[0]}-cin{c[1]}-cout{c[2]}-K{c[3]}" for c in DENSE])
def test_densest_graph_vs_float64(case):
    """E_max edges (duplicates allowed) fill the layout at T = 12: `dcrnn_seq_supported` holds and the kernel runs; one edge more and
    it is refused."""
    n, cin, cout, K, route = case
    E = _max_edges(n, cin, cout, K, SUPPORT_T)
    m = _dcrnn_model(cin, cout, K, seed=n)
    errs = []
    plan, ei, ew = _plan_of(m, _edges(n, E, 1), n)
    assert _nnz(plan, False) == (E, E)
    _case(errs, m, plan, ei, ew, 2, SUPPORT_T, n, ("densest", n, E), route=route)
    plan, _, _ = _plan_of(m, _edges(n, E + 1, 2), n)
    e = Expect(plan, cin, cout, K, 2, SUPPORT_T, tc=False)
    assert e.tmax < SUPPORT_T and e.fwd is None
    assert not errs, errs[:6]


# ---- 4. K = 2 at 32 channels past the graph images: the persistent backward behind the FFMA stash, and past it ----------------------
E_DENSE = E_IMAGE + 4                            # four edges past the densest graph with an image at 207 nodes: a T = 12 layout at cin 1
WIDE = [  # (N, graph, cins, backward route)
    (207, ("edges", E_DENSE), (1,), ("bwd", "pair", "global")),
    (207, ("long", 509), (1, 2, 3, 4), ("bwd", "pair", "staged")),
    (208, ("random",), (1, 2, 3, 4), ("bwd", "pair", "staged")),
    (208, ("edges", 2090), (2,), ("bwd", "pair", "staged")),
    (208, ("edges", 2091), (1,), ("bwd", "pair", "global")),
    (216, ("edges", 435), (3,), ("bwd", "pair", "staged")),
    (216, ("edges", 436), (4,), ("bwd", "pair", "global")),
    (217, ("random",), (3, 4), ("bwd", "per-step")),
    (217, ("random",), (1, 2), ("bwd", "pair", "staged")),
    (224, ("random",), (2,), ("bwd", "pair", "global")),
    (225, ("ring",), (1,), ("bwd", "pair", "staged")),
    (225, ("edges", 226), (2,), ("bwd", "pair", "global")),
    (228, ("edges", 4 * 228), (1, 2), ("bwd", "pair", "global")),
    (232, ("random",), (1, 2), ("bwd", "pair", "global")),
    (233, ("random",), (1, 2), ("bwd", "per-step")),
    (256, ("random",), (1, 4), ("bwd", "per-step")),
]


def _wide_graph(n, g):
    if g[0] == "long":
        return _long_row(n, g[1]), None
    if g[0] == "edges":
        return geo_graph("edges", n, g[1]), None
    return make_graph(g[0], n), g[0]


@pytest.mark.parametrize("case", WIDE, ids=[f"N{c[0]}-{'-'.join(map(str, c[1]))}-cin{''.join(map(str, c[2]))}-{'-'.join(c[3][1:])}"
                                            for c in WIDE])
def test_k2_wide_state_past_the_images_vs_float64(case):
    """BatchedDCRNN(cin, 32, 2) on graphs the wgmma kernel cannot take: no graph image at 207 nodes (too dense, or a row of 509
    entries), 208-256 nodes.  Inference, then training with the persistent backward (staged or global graph; CTA pair and one CTA bit
    for bit) or, past `fits_one_sm`, the per-step backward; the module routes the same call to the FFMA kernel."""
    n, g, cins, route = case
    graph, kind = _wide_graph(n, g)
    errs = []
    for cin in cins:
        m = _dcrnn_model(cin, 32, 2, seed=n + cin)
        plan, ei, ew = _plan_of(m, graph, n, kind)
        e = Expect(plan, cin, 32, 2, 3, 4)
        assert not e.tc and e.fwd is not None, (n, g, cin, e.label())
        _case(errs, m, plan, ei, ew, 3, 4, n * cin, ("wide", n, g, cin), h0=cin % 2 == 1, tc=True, route=route)
        if e.tmax >= SUPPORT_T:                  # else (cin 4 from 207 nodes) `dcrnn_seq_supported` is false and the module goes elsewhere
            X = torch.randn(2, 3, n, cin, device=DEV)
            with torch.no_grad(), _counted() as c:
                m(X, ei, ew)
            _assert_fwd(c, Expect(plan, cin, 32, 2, 2, 3), plain_loads(n, cin, 3, X, False), ("module", n, g, cin))
    assert not errs, errs[:6]


# ---- 5. the window length past the X buffer ------------------------------------------------------------------------------------------
TLIMIT = [(228, 2, 32, 2), (201, 3, 16, 3)]      # (N, cin, cout, K); 4N edges


@pytest.mark.parametrize("case", TLIMIT, ids=[f"N{c[0]}-cin{c[1]}-cout{c[2]}-K{c[3]}" for c in TLIMIT])
def test_window_length_at_and_past_the_x_buffer_vs_float64(case):
    """At the mirror's largest T the kernel runs (at 228 nodes, cin 2, K 2: 17); at T + 1 `dcrnn_seq_fwd` raises StmpUnsupported and
    BatchedDCRNN, for inference and training, lands on the tiled path -- still held to float64."""
    n, cin, cout, K = case
    m = _dcrnn_model(cin, cout, K, seed=n)
    plan, ei, ew = _plan_of(m, geo_graph("edges", n, 4 * n), n)
    tmax = max_T(n, _nnz(plan, False), cin, cout, K)
    assert tmax >= SUPPORT_T and (n != 228 or tmax == 17)
    errs = []
    _case(errs, m, plan, ei, ew, 2, tmax, n, ("T limit", n, tmax), train=False)
    T = tmax + 1
    gen = torch.Generator(device=DEV).manual_seed(T)
    X = torch.randn(2, T, n, cin, device=DEV, generator=gen)
    wgt = torch.randn(2, T, n, cout, device=DEV, generator=gen)
    assert Expect(plan, cin, cout, K, 2, T).fwd is None
    with pytest.raises(_lib.StmpUnsupported):
        ops.dcrnn_seq_fwd(plan, X, *m._params(), K)
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    x64 = X.double().requires_grad_(True)
    with _float64():
        out64 = R.batched_dcrnn(p64, x64, ei, ew.double())
    g64 = _loss_grads([out64], [wgt.double()], [x64] + [p64[k] for k in names])
    with torch.no_grad(), _counted() as c:
        inf = m(X, ei, ew)
    xf = X.clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    with _counted() as ct:
        out = m(xf, ei, ew)
        gf = _loss_grads([out], [wgt], [xf] + params)
    for cc in (c, ct):
        assert not [k for k in cc if k.startswith(("k_dcrnn_seq", "k_dcrnn_bwd", "k_gru_bwd", "k_dcrnn_rows", "k_dcrnn_nrows"))], cc
        assert cc.get("k_spmm", 0) > 0, cc
    LAUNCHED.add(("tiled",))
    with torch.no_grad():
        out32 = _tiled(m, plan, X)
    x32 = X.clone().requires_grad_(True)
    m.zero_grad(set_to_none=True)
    g32 = _loss_grads([_tiled(m, plan, x32)], [wgt], [x32] + params)
    what = ("past the X buffer", n, T)
    _check_err(errs, FAM + "tiled route", inf, out32, out64, what + ("out, no_grad",))
    _check_err(errs, FAM + "tiled route", out, out32, out64, what + ("out",))
    for label, got, r32, r64 in zip(["dX"] + names, gf, g32, g64):
        _check_err(errs, FAM + "tiled route", got, r32, r64, what + (label,))
    assert not errs, errs[:6]


# ---- 6. windows: CTAs that reuse their first X buffer, the indexed entry, misaligned X, a state per window, the cell -----------------
WINDOW_B = ("1", "SMs", "SMs+1", "3SMs+1")
WINDOW_LOADS = {"tma": (40, 2), "plain": (41, 1)}       # (N, cin): T N cin = 240 (whole 16-byte windows) / 123 at T = 3


def _windows(name):
    s = _sms()
    return {"1": 1, "SMs": s, "SMs+1": s + 1, "3SMs+1": 3 * s + 1}[name]


@pytest.mark.parametrize("b,load", [(b, ld) for b in WINDOW_B for ld in WINDOW_LOADS], ids=[f"B{b}-{ld}" for b in WINDOW_B for ld in WINDOW_LOADS])
def test_windows_and_buffer_reuse_vs_float64(b, load):
    """B windows with a state per window: at 3 SMs + 1 CTA 0 runs four windows and waits on its first TMA buffer a second time (the
    mbarrier's second phase).  The first, last and every SMs-th window equal the same window run alone bit for bit; those windows are
    held to float64."""
    n, cin = WINDOW_LOADS[load]
    cout, K, T = 16, 3, 3
    B = _windows(b)
    m = _dcrnn_model(cin, cout, K, seed=B)
    plan, ei, ew = _plan_of(m, make_graph("mod4", n), n, "mod4")
    e = Expect(plan, cin, cout, K, B, T)
    gen = torch.Generator(device=DEV).manual_seed(B)
    X = torch.randn(B, T, n, cin, device=DEV, generator=gen)
    H0 = 0.5 * torch.randn(B, n, cout, device=DEV, generator=gen)
    assert plain_loads(n, cin, T, X, False) == (load == "plain")
    with torch.no_grad(), _counted() as c:
        out = ops.dcrnn_seq_fwd(plan, X, *m._params(), K, h0=H0)
    _assert_fwd(c, e, load == "plain", ("windows", B))
    pick = sorted({0, B - 1} | set(range(0, B, _sms())))
    with torch.no_grad():
        for i in pick:
            alone = ops.dcrnn_seq_fwd(plan, X[i:i + 1], *m._params(), K, h0=H0[i:i + 1])
            assert torch.equal(alone[0], out[i]), ("window", i, "of", B, "differs from the same window run alone")
        out32 = _tiled(m, plan, X[pick], H0[pick])
    sd64 = {k: v.detach().double() for k, v in m.state_dict().items()}
    with _float64(), torch.no_grad():
        out64 = _oracle_seq(sd64, X[pick].double(), ei, ew.double(), H0[pick].double())
    errs = []
    _check_err(errs, FAM + "forward", out[pick], out32, out64, ("windows", B, load, e.label()))
    assert not errs, errs


INDEXED = {"tma": (60, 2, 32, 3), "plain": (61, 3, 16, 4)}      # (N, cin, cout, K): N cin = 120 / 183


@pytest.mark.parametrize("load", list(INDEXED))
def test_forward_indexed_vs_gathered_windows(load):
    """`forward_indexed` reads overlapping windows in place from the series (win_start): equal bit for bit to `forward` on the
    gathered windows, TMA loads when a window row is whole 16-byte units (N cin % 4 == 0), plain loads otherwise; then the same from a
    series slice whose data pointer is 4 bytes past a 16-byte boundary (plain loads whatever N cin is)."""
    n, cin, cout, K = INDEXED[load]
    T, B = 12, 2 * _sms() + 3
    m = _dcrnn_model(cin, cout, K, seed=n)
    plan, ei, ew = _plan_of(m, make_graph("hubs", n), n, "hubs")
    flat = torch.randn(1 + 80 * n * cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(n))
    series = flat[:-1].view(80, n, cin)
    starts = torch.randint(0, 80 - T + 1, (B,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    starts[:4] = torch.tensor([0, 68, 3, 3])                     # the last window, and one repeated
    e = Expect(plan, cin, cout, K, B, T)
    errs, got_aligned = [], None
    for src, what in ((series, "aligned"), (flat[1:].view(80, n, cin), "series 4 bytes past 16")):
        plain = plain_loads(n, cin, T, src, True)
        assert plain == (load == "plain" or what != "aligned")
        with torch.no_grad():
            with _counted() as c:
                got = m.forward_indexed(src, starts, T, ei, ew)
            _assert_fwd(c, e, plain, ("indexed", load, what))
            X = ops.window_gather(src, starts, T, with_target=False)
            with _counted() as c:
                mat = m(X, ei, ew)
            _assert_fwd(c, e, plain_loads(n, cin, T, X, False), ("gathered", load, what))
        assert torch.equal(got, mat), ("indexed windows differ from the gathered ones", load, what)
        got_aligned = got if got_aligned is None else got_aligned
    X = ops.window_gather(series, starts[:3], T, with_target=False)
    with torch.no_grad():
        out32 = _tiled(m, plan, X)
    with _float64(), torch.no_grad():
        out64 = R.batched_dcrnn({k: v.double() for k, v in m.state_dict().items()}, X.double(), ei, ew.double())
    _check_err(errs, FAM + "forward", got_aligned[:3], out32, out64, ("indexed", load, e.label()))
    assert not errs, errs


def test_misaligned_windows_take_plain_loads():
    """X (B, T, N, cin) contiguous but 4 bytes past a 16-byte boundary, with T N cin % 4 == 0: plain loads, bit for bit the aligned
    result; inference and the training forward."""
    n, cin, cout, K, B, T = 50, 2, 32, 4, 3, 4
    m = _dcrnn_model(cin, cout, K, seed=5)
    plan, ei, ew = _plan_of(m, make_graph("lonely", n), n, "lonely")
    flat = torch.randn(1 + B * T * n * cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    Xa = flat[:-1].view(B, T, n, cin).clone()
    Xm = flat[1:].view(B, T, n, cin)
    Xm.copy_(Xa)
    e = Expect(plan, cin, cout, K, B, T)
    assert not plain_loads(n, cin, T, Xa, False) and plain_loads(n, cin, T, Xm, False)
    outs = []
    for X, plain in ((Xa, False), (Xm, True)):
        with torch.no_grad(), _counted() as c:
            outs.append(ops.dcrnn_seq_fwd(plan, X, *m._params(), K))
        _assert_fwd(c, e, plain, ("misaligned", plain))
        with _counted() as c:
            outs.append(_DcrnnSeqFn.apply(X.requires_grad_(False), None, *m._params(), plan, K, None).detach())
        _assert_fwd(c, e, plain, ("misaligned, training forward", plain))
    assert all(torch.equal(outs[0], o) for o in outs[1:])


CELLS = [(3, 16, 4, "mod4"), (2, 32, 1, "hubs"), (1, 32, 3, "lonely")]


@pytest.mark.parametrize("cell", CELLS, ids=[f"cin{c[0]}-cout{c[1]}-K{c[2]}-{c[3]}" for c in CELLS])
def test_dcrnn_cell_vs_float64(cell):
    """The DCRNN cell (unbatched semantics: the reference's dense-adjacency degrees) with H given and not, inference and training,
    against `R.dcrnn_cell`: one window, one step, the per-step backward."""
    cin, cout, K, kind = cell
    n = 70
    g = make_graph(kind, n)
    ei, ew = _tensors(g)
    torch.manual_seed(cin + cout + K)
    m = DCRNN(cin, cout, K).to(DEV)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if name.endswith(".bias"):
                p.normal_(0, 0.1)
    plan = m._plan(ei, ew, n)
    check_family(kind, n, g, plan, cheb=False)
    e = Expect(plan, cin, cout, K, 1, 1)
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    errs = []
    for given in (True, False):
        what = ("cell", kind, cin, cout, K, given, e.label())
        gen = torch.Generator(device=DEV).manual_seed(K + given)
        X = torch.randn(n, cin, device=DEV, generator=gen)
        H = 0.5 * torch.randn(n, cout, device=DEV, generator=gen) if given else None
        wgt = torch.randn(n, cout, device=DEV, generator=gen)
        p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
        x64 = X.double().requires_grad_(True)
        h64 = None if H is None else H.double().requires_grad_(True)
        with _float64():
            o64 = R.dcrnn_cell(p64, x64, ei, ew.double(), h64)
        g64 = _loss_grads([o64], [wgt.double()], [x64, h64] + [p64[k] for k in names])
        x32 = X.clone().requires_grad_(True)
        h32 = None if H is None else H.clone().requires_grad_(True)
        m._fused_training = False
        m.zero_grad(set_to_none=True)
        try:
            o32 = m(x32, ei, ew, h32)
        finally:
            m._fused_training = True
        g32 = _loss_grads([o32], [wgt], [x32, h32] + params)
        with torch.no_grad(), _counted() as c:
            inf = m(X, ei, ew, H)
        _assert_fwd(c, e, plain_loads(n, cin, 1, X, False), what)
        xf = X.clone().requires_grad_(True)
        hf = None if H is None else H.clone().requires_grad_(True)
        m.zero_grad(set_to_none=True)
        with _counted() as cf:
            of = m(xf, ei, ew, hf)
        with _counted() as cb:
            gf = _loss_grads([of], [wgt], [xf, hf] + params)
        _assert_fwd(cf, e, plain_loads(n, cin, 1, X, False), what)
        _assert_bwd(cb, e, what)
        assert torch.equal(of.detach(), inf), what
        _check_err(errs, FAM + "forward", inf, o32, o64, what + ("out",))
        for i, (label, got, r32, r64) in enumerate(zip(["dX", "dH"] + names, gf, g32, g64)):
            if i == 1 and H is None:
                assert got is None, what
                continue
            _check_err(errs, FAM + "per-step backward", got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (label,))
    assert not errs, errs[:6]


# ---- 7. the per-step backward: every K at 16 and 32 channels ----------------------------------------------------------------------
PER_STEP = [(cout, K) for cout in (16, 32) for K in (1, 2, 3, 4)]


@pytest.mark.parametrize("cout,K", PER_STEP, ids=[f"cout{co}-K{K}" for co, K in PER_STEP])
def test_per_step_backward_vs_float64(cout, K):
    """`_DcrnnSeqFn.backward`'s per-step branch behind the FFMA stash: dX and H0 wanted, then neither.  K = 2 at 32 channels has the
    persistent backward below 233 nodes, so it runs at 233 and 256 nodes; the others at 90 nodes, on a graph with every degree
    residue."""
    errs = []
    for j, n in enumerate((233, 256) if (cout, K) == (32, 2) else (90,)):
        cin = 1 + (K + j) % 2 if n > 216 else 1 + (K + cout // 16) % 4
        m = _dcrnn_model(cin, cout, K, seed=10 * K + cout + j)
        plan, ei, ew = _plan_of(m, make_graph("mod4", n, seed=j), n, "mod4")
        for full in (True, False):
            _case(errs, m, plan, ei, ew, 3, 4, n + K + full, ("per-step", n, cin, cout, K, full), h0=full, want_dx=full,
                  route=("bwd", "per-step"))
    assert not errs, errs[:6]


def test_cfg2_shape_with_the_persistent_backward_switched_off_vs_float64():
    """BatchedDCRNN(2, 32, 2) at the benchmark's window length (T = 12) on 207 nodes without a graph image: `fused_backward = False`
    sends the step the persistent kernel would take through the per-step branch; both are held to float64."""
    n, cin = 207, 2
    m = _dcrnn_model(cin, 32, 2, seed=2)
    plan, ei, ew = _plan_of(m, _long_row(n, 509), n)
    errs = []
    for fused in (False, True):
        route = ("bwd", "pair", "staged") if fused else ("bwd", "per-step")
        _case(errs, m, plan, ei, ew, 2, 12, 22, ("cfg2 shape", fused), tc=True, fused_bwd=fused, route=route)
    assert not errs, errs[:6]


# ---- 8. the reference's example model ------------------------------------------------------------------------------------------------
def test_reference_example_model_on_chickenpox_vs_float64():
    """examples/recurrent/dcrnn_example.py: DCRNN(4, 32, 1) -> ReLU -> Linear(32, 1) on the chickenpox graph, H = None per snapshot,
    the MSE summed over 6 snapshots: every parameter gradient against float64 through the FFMA kernel and the per-step backward."""
    ei, ew, X, Y = chickenpox_train_split()
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X[:6].to(DEV), Y[:6].to(DEV)
    n = X.shape[1]
    torch.manual_seed(0)
    rec, lin = DCRNN(4, 32, 1).to(DEV), torch.nn.Linear(32, 1).to(DEV)
    with torch.no_grad():
        for name, p in rec.named_parameters():
            if name.endswith(".bias"):
                p.normal_(0, 0.1)
    plan = rec._plan(ei, ew, n)
    e = Expect(plan, 4, 32, 1, 1, 1)
    params = list(rec.parameters()) + list(lin.parameters())
    names = [k for k, _ in rec.named_parameters()] + ["linear." + k for k, _ in lin.named_parameters()]

    def loss(cell, linear):
        return sum(((linear(torch.relu(cell(X[s]))).squeeze(-1) - Y[s]) ** 2).mean() for s in range(X.shape[0]))

    p64 = {k: v.detach().double().requires_grad_(True) for k, v in rec.state_dict().items()}
    l64 = {k: v.detach().double().requires_grad_(True) for k, v in lin.state_dict().items()}
    with _float64():
        cost64 = loss(lambda x: R.dcrnn_cell(p64, x.double(), ei, ew.double()),
                      lambda h: h @ l64["weight"].T + l64["bias"])
        g64 = torch.autograd.grad(cost64, list(p64.values()) + list(l64.values()))
    rec._fused_training = False
    try:
        cost32 = loss(lambda x: rec(x, ei, ew), lin)
        g32 = torch.autograd.grad(cost32, params)
    finally:
        rec._fused_training = True
    with _counted() as c:
        cost = loss(lambda x: rec(x, ei, ew), lin)
        gf = torch.autograd.grad(cost, params)
    assert c.get("k_dcrnn_seq") == c.get("k_dcrnn_seq[<32,1,8>]") == c.get("k_gru_bwd_zr") == X.shape[0], c
    assert e.fwd == (32, 1, 8) and not e.persistent and "k_dcrnn_bwd_seq" not in c and "k_spmm" not in c
    errs = []
    _check_err(errs, FAM + "example model", cost, cost32, cost64, ("chickenpox", "cost"))
    for label, got, r32, r64 in zip(names, gf, g32, g64):
        _check_err(errs, FAM + "example model", got, r32, r64, ("chickenpox", label))
    assert not errs, errs
