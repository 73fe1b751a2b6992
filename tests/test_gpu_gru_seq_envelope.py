"""The generic graph-GRU sequence kernels (`stmp_gru_seq_fwd` and `stmp_gru_bwd_*`: `k_dcrnn_seq_tc` / `k_dcrnn_seq_rf`,
`k_gru_pack_bwd_weights`, `k_gru_bwd_basis`, `k_gru_bwd_seq`, `k_dcrnn_wgrad_tc`, `k_gru_wgrad_reduce`; DESIGN §4, §4h) against float64
across their envelope: every plan flavor and operator count they serve (Chebyshev K = 1, 2 with `sym`, `rw` and None, given and
default lambda_max; GCN; DConv with one and two operators), cin 1..4 with and without bias, node counts on both sides of the
backward's CTA-pair threshold (16), the 64 / 128-row tiles and the forward's pair threshold (128), up to the 207-node limit and past
it, windows on both sides of SMs / 2 and SMs (the forward's persistent loop), 65 536 windows, step counts whose T * cin crosses the
workspace pitch, an initial state that is absent, per window or shared, every subset of requested gradients, and the GConvGRU module.

A Python mirror of the launch logic (`mirror`, from `tc_launch_params` / `tc_fits` in dcrnn_seq_tc.cu and `seq_impl` / `graph_in_smem`
/ `fits_one_sm` in dcrnn_bwd.cu) predicts for every call which variant serves it -- forward CTA pair (N > 128 and 2 B <= SMs), one CTA,
or one persistent CTA per SM (B > SMs); backward CTA pair (2 B <= SMs and N >= 16) or one CTA, with the transposed operators staged in
shared memory or read from the global CSR -- and every case asserts that `ops.gru_seq_supported` / `gru_bwd_supported` and the path
counters agree with it.  `_report` checks at the end of the module that every reachable variant ran.  The backward's global-CSR
variant at one operator cannot be reached through `ops.gru_seq_train` (`test_one_operator_global_csr_backward_from_a_float64_stash`
computes why), so that test drives it through `ops.gru_bwd_basis` / `gru_bwd_seq` / `gru_bwd_wgrad` on a float64 stash.

Numerical criterion (the one of test_gpu_rows_envelope.py, whose helpers this file imports): against float64, the fused path's largest
error stays within 4x that of the fp32 op-for-op path plus 2^-20 of the tensor's scale -- for the output, dX, dH0, dwcat and dbcat.
The fp32 op-for-op path is `_restated` of test_gpu_gconv_gru_train.py over `ops.spmm`; the float64 reference is the same recurrence
on dense float64 operators built from edge_index / edge_weight with the oracle's normalization (`oracle.pyg.cheb_norm`, `gcn_norm`,
`oracle.recurrent.dconv_operators`), never from the plan's fp32 values.  `test_plan_operators_are_the_oracle_rounded` checks
separately that each plan operator is the oracle's rounded to fp32.

Largest error ratios of one run on an H100 (80 GB HBM3, 700 W power limit), as printed by `_report` -- observations, not guarantees.
`e / e32` is taken over the comparisons whose error exceeds the 2^-20 floor; `used` is the largest fraction of the allowance
4 e32 + 2^-20 scale that any comparison consumed (two measured departures from 4x are allowed more, see `_allow`; L = D - A below
its default lambda_max is held step by step, see `_op_scale`):
    forward, n_ops 0 / 1 / 2                     e / e32  0.00 / 2.25 / 3.62   used 0.26 / 0.46 / 0.76
    backward, CTA pair: no graph / staged / global          0.00 / 5.69 / 0.00        0.37 / 1.37 / 0.38   (5.69: T = 40, dH0, allowed 8x)
    backward, one CTA: no graph / staged / global           10.58 / 11.69 / 3.37      1.44 / 1.66 / 0.49   (B = 2 SMs + 5, dwcat, allowed 16x)
    backward kernels on a float64 stash (all variants)      2.97                      0.48
    forward, one step from the float64 state                 0.00                      0.68   (floor scaled by the operands)
    weight-gradient contraction alone                        7.83                      1.14   (111 366 rows, dwcat, allowed 16x)
    GConvGRU module                                          3.63                      0.51
The whole file (77 tests) ran in 37 s there.
"""
import contextlib
import functools
import itertools

import numpy as np
import pytest
import torch

from oracle import pyg as P
from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN, GConvGRU
from pytorch_geometric_temporal_b200.plan import GraphPlan
from test_gpu_gconv_gru_train import _restated
from test_gpu_graph_geometry import BWD_SMEM, IMG_MAX_N, TC_SMEM, _option, bwd_staged, image_fits, ncol_of
from test_gpu_graph_geometry import make_graph as make_sized_graph
from test_gpu_rows_envelope import WORST, _check_err, _counted, _float64, _loss_grads, make_graph
from test_row_image_cpu import build_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
FAM = "gru one-SM: "                              # prefix of this file's families in WORST

# ---- the mirror of the launch logic --------------------------------------------------------------------------------------------------
RI_BUDGET = TC_SMEM - (4 * 96 * 128 + 2 * 256 * 32 * 4 + 96 * 4 + 8)   # rf_layout: B panels, two gather buffers, biases, mbarrier
BWD_THREADS = 512
WATCH = ("k_dcrnn_seq_tc", "k_dcrnn_seq_tc[cluster2]", "k_dcrnn_seq", "k_gru_pack_bwd_weights", "k_gru_bwd_basis", "k_gru_bwd_seq",
         "k_gru_bwd_seq[cluster2]", "k_gru_bwd_seq[graph-global]", "k_dcrnn_wgrad_tc", "k_gru_wgrad_reduce", "k_spmm")


@functools.lru_cache(maxsize=None)
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _csr(plan, op):
    rp, col, val, _ = plan.export(op)
    return rp.cpu().numpy(), col.cpu().numpy(), val.cpu().numpy()


def _fits_one_sm(n, cin, n_ops):
    """dcrnn_bwd.cu fits_one_sm: the GEMM tiles fit the block, the per-window buffers its shared memory, the basis kernel's copies 100 KB."""
    ncol, rg = ncol_of(cin, n_ops), (n + 7) // 8
    base = 4 * (3 * 32 * ncol + rg * 8 * ncol + 2 * 32 * (rg * 8 + 4) + n * 36)
    return rg * (ncol // 8) <= BWD_THREADS and base <= BWD_SMEM and 8 * n * (cin + 32) <= 100 * 1024


@functools.lru_cache(maxsize=None)
def _images(plan, n_ops):
    """tc_fits: both shared-memory images of the first n_ops operators exist (the graph image of the pair, the row image of one CTA)."""
    n = plan.num_nodes
    if not 1 <= n <= IMG_MAX_N:
        return False
    if n_ops == 0:
        return True
    ri = build_ref(n, [_csr(plan, op) for op in range(n_ops)])
    return image_fits(n, n_ops, sum(plan.nnz(op) for op in range(n_ops))) and len(ri) <= RI_BUDGET


def mirror(plan, n_ops, cin, B, fwd_split=True, bwd_split=True):
    """(forward supported, forward variant, backward supported, backward variant, graph) for a call of B windows."""
    n, S = plan.num_nodes, _sms()
    ok = 1 <= cin <= 4 and 0 <= n_ops <= min(2, plan.n_ops)
    fwd = "pair" if fwd_split and n > 128 and 2 * B <= S else ("persistent" if B > S else "one")
    bwd = "pair" if bwd_split and 2 * B <= S and n >= 16 else "one"
    graph = "none" if n_ops == 0 else ("staged" if bwd_staged(n, cin, [plan.nnz(op) for op in range(n_ops)]) else "global")
    return ok and _images(plan, n_ops), fwd, ok and _fits_one_sm(n, cin, n_ops), bwd, graph


def _check_support(plan, n_ops, cin):
    fwd_ok, _, bwd_ok, _, _ = mirror(plan, n_ops, cin, 1)
    assert ops.gru_seq_supported(plan, n_ops, cin, 32) == fwd_ok, (plan.num_nodes, n_ops, cin)
    assert ops.gru_bwd_supported(plan, n_ops, cin, 32) == bwd_ok, (plan.num_nodes, n_ops, cin)
    return fwd_ok, bwd_ok


LAUNCHED = set()
REACHABLE = ({("fwd", v, cin, k) for v in ("pair", "one", "persistent") for cin in (1, 2, 3, 4) for k in (0, 1, 2)}
             | {("bwd", v, g, cin, k) for v in ("pair", "one") for cin in (1, 2, 3, 4) for k in (0, 1, 2)
                for g in (("none",) if k == 0 else ("staged", "global"))})


def _expect(m, fwd=True, bwd=False, wgrad=False):
    _, fv, _, bv, graph = m
    want = {}
    if fwd:
        want.update({"k_dcrnn_seq_tc": 1, "k_dcrnn_seq_tc[cluster2]": int(fv == "pair")})
    if bwd:
        want.update({"k_gru_pack_bwd_weights": 1, "k_gru_bwd_basis": 1, "k_gru_bwd_seq": 1, "k_gru_bwd_seq[cluster2]": int(bv == "pair"),
                     "k_gru_bwd_seq[graph-global]": int(graph == "global"), "k_dcrnn_wgrad_tc": int(wgrad),
                     "k_gru_wgrad_reduce": int(wgrad)})
    return {k: v for k, v in want.items() if v}


def _assert_launches(c, want, what):
    got = {k: v for k, v in c.items() if k in WATCH}
    assert got == want, (what, got, want)


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    failed_before = request.session.testsfailed
    yield
    for fam, (ratio, used, what) in sorted(WORST.items()):
        if fam.startswith(FAM):
            print(f"\ngru envelope: {fam[len(FAM):]}: largest e / e32 = {ratio:.2f}, largest used fraction of the allowance = {used:.2f} at {what}")
    # checked when every test of this module was selected and none of them failed (a failing case stops before its later launches)
    here = {it.originalname for it in request.session.items if it.module is request.module}
    every = {k for k, v in vars(request.module).items() if k.startswith("test_") and callable(v)}
    failed_here = request.session.testsfailed - failed_before
    print(f"gru envelope: variant check {'runs' if here == every and not failed_here else 'skipped'} "
          f"({len(here)} of {len(every)} tests selected, {failed_here} failed here); {len(LAUNCHED)} of {len(REACHABLE)} variants ran")
    if here == every and not failed_here:
        assert LAUNCHED == REACHABLE, ("variants never launched", sorted(REACHABLE - LAUNCHED))


# ---- plans and their float64 operators -----------------------------------------------------------------------------------------------
# (name, flavor, n_ops, keyword arguments): Chebyshev K = 1 (n_ops = 0) and K = 2 (n_ops = 1) per normalization and lambda_max,
# GCN (improved, self loops, unweighted), DConv with one and two operators
PLANS = ([(f"cheb{k + 1}-{norm}-{'lam' if lam else 'dflt'}", "cheb", k, dict(norm=norm, lam=lam))
          for k in (0, 1) for norm in ("sym", "rw", None) for lam in (None, 1.7)]
         + [("gcn", "gcn", 1, dict(improved=False, loops=True, weighted=True)),
            ("gcn-improved-unweighted", "gcn", 1, dict(improved=True, loops=True, weighted=False)),
            ("gcn-no-loops", "gcn", 1, dict(improved=False, loops=False, weighted=True)),
            ("dconv1", "dconv", 1, {}), ("dconv2", "dconv", 2, {})])


def _dense(ei, w, n):
    """The operator y[dst] += w x[src] of an edge list as a dense float64 matrix (duplicates summed)."""
    A = torch.zeros(n, n, dtype=torch.float64, device=DEV)
    A.index_put_((ei[1], ei[0]), w.double(), accumulate=True)
    return A


def build(flavor, g, n, norm=None, lam=None, improved=False, loops=True, weighted=True):
    """(plan, [dense float64 operators]) of graph g; the operators come from the oracle's normalization of edge_index / edge_weight."""
    src, dst, w = g
    ei = torch.from_numpy(np.stack([src, dst])).to(DEV)
    ew = torch.from_numpy(w).to(DEV)
    with _float64():
        if flavor == "cheb":
            plan = GraphPlan(_lib.FLAVOR_CHEB, ei, ew, n, norm, lam)
            loose = src != dst                     # L = D - A below its default lambda_max, 2 max(degree): see _op_scale
            plan.amplifying = norm is None and lam is not None and lam < 2 * np.bincount(src[loose], w[loose], n).max(initial=0)
            ops64 = [_dense(*P.cheb_norm(ei, n, ew.double(), norm, lam, dtype=torch.float64), n)]
        elif flavor == "gcn":
            flags = (_lib.GCN_IMPROVED if improved else 0) | (0 if loops else _lib.GCN_NO_SELF_LOOPS)
            plan = GraphPlan(_lib.FLAVOR_GCN, ei, ew if weighted else None, n, flags=flags)
            ops64 = [_dense(*P.gcn_norm(ei, ew.double() if weighted else None, n, improved, loops, dtype=torch.float64), n)]
        else:
            plan = GraphPlan(_lib.FLAVOR_DCONV, ei, ew, n, flags=_lib.DCONV_ALLOW_DUPLICATES)
            ei_o, n_o, ei_i, n_i = R.dconv_operators(ei, ew.double(), batched=True, num_nodes=n)
            ops64 = [_dense(ei_o, n_o, n), _dense(ei_i, n_i, n)]
    plan.amplifying = getattr(plan, "amplifying", False)
    return plan, ops64


def _plan_dense(plan, op):
    rp, col, val, _ = plan.export(op)
    n = plan.num_nodes
    rows = torch.repeat_interleave(torch.arange(n, device=DEV), (rp[1:] - rp[:-1]).long())
    A = torch.zeros(n, n, dtype=torch.float64, device=DEV)
    A.index_put_((rows, col.long()), val.double(), accumulate=True)
    return A


# (N, graph kind): hubs, every in- and out-degree residue mod 4, duplicates (DConv only), a row with nothing but a self loop, a node
# without out-edges, the ring, random graphs
GEOS = [(1, "ring"), (2, "random"), (15, "mod4"), (16, "hubs"), (63, "sink"), (64, "lonely"), (65, "mod4_out"), (127, "dups"),
        (128, "hubs"), (129, "random"), (206, "mod4"), (207, "hubs")]


@functools.lru_cache(maxsize=None)
def _graph(kind, n):
    return make_graph(kind, n)


# ---- one case ------------------------------------------------------------------------------------------------------------------------
def _weights(n_ops, cin, bias, gen):
    """(wcat (96, 112), bcat (96,)) in the forward's layout, columns H | Op0 H | Op1 H | X | Op0 X | Op1 X | pad; zeros where the layout
    has no column."""
    wcat = torch.zeros(96, 112, device=DEV)
    for k in range(n_ops + 1):
        wcat[:, 32 * k:32 * k + 32] = torch.randn(96, 32, device=DEV, generator=gen) * 0.15
        wcat[:, 96 + 4 * k:96 + 4 * k + cin] = torch.randn(96, cin, device=DEV, generator=gen) * 0.3
    bcat = torch.randn(96, device=DEV, generator=gen) * 0.1 if bias else torch.zeros(96, device=DEV)
    return wcat, bcat


def _live(n_ops, cin):
    live = torch.zeros(96, 112, dtype=torch.bool, device=DEV)
    for k in range(n_ops + 1):
        live[:, 32 * k:32 * k + 32] = True
        live[:, 96 + 4 * k:96 + 4 * k + cin] = True
    return live


def _inputs(plan, n_ops, cin, B, T, seed, h0, bias):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    N = plan.num_nodes
    wcat, bcat = _weights(n_ops, cin, bias, gen)
    x = torch.randn(B, T, N, cin, device=DEV, generator=gen)
    H0 = None if h0 == "none" else 0.5 * torch.randn(B, N, 32, device=DEV, generator=gen)
    wgt = torch.randn(B, T, N, 32, device=DEV, generator=gen)
    return x, H0, wcat, bcat, wgt


def _leaves(cast, x, H0, wcat, bcat, want, bias):
    return [cast(x).requires_grad_("x" in want), None if H0 is None else cast(H0).requires_grad_("h0" in want),
            cast(wcat).requires_grad_("w" in want), cast(bcat).requires_grad_("w" in want and bias) if bias else None]


def _refs(plan, ops64, n_ops, x, H0, wcat, bcat, wgt, want, bias):
    """(float64 and fp32 op-for-op) lists [out, dX, dH0, dwcat, dbcat] (None where not wanted) of the mean loss <out, wgt>."""
    res = []
    for cast, spmm in ((lambda t: t.detach().double(), lambda k, t: ops64[k] @ t), (lambda t: t.detach().clone(), None)):
        lv = _leaves(cast, x, H0, wcat, bcat, want, bias)
        with (_float64() if spmm else contextlib.nullcontext()):
            out = _restated(plan, n_ops, lv[0], lv[1], lv[2], lv[3] if bias else cast(bcat), spmm=spmm)
        grads = _loss_grads([out], [cast(wgt)], lv) if want else [None] * 4
        res.append([out.detach()] + grads)
    return res


def _fused(plan, n_ops, x, H0, wcat, bcat, wgt, want, bias, wimage=False):
    lv = _leaves(lambda t: t.detach().clone(), x, H0, wcat, bcat, want, bias)
    spec = [("w", 0, 96, 0, 112)] + ([("b", 0, 96)] if bias else [])
    params = [lv[2]] + ([lv[3]] if bias else [])
    img = ops.gru_weight_image(wcat, bcat) if wimage else None
    out = ops.gru_seq_train(plan, n_ops, lv[0], lv[1], wcat, bcat, img, spec, params)
    assert out.requires_grad == bool(want)
    grads = _loss_grads([out], [wgt], lv) if want else [None] * 4
    return [out.detach()] + grads


def _run(errs, plan, ops64, n_ops, cin, B, T, seed, what, h0="window", want=("x", "h0", "w"), bias=True, wimage=False):
    """Inference and one training step of the fused kernels at (B, T) on `plan` against float64: the launches the mirror predicts,
    training output bit-identical to inference, unwanted gradients None, dead weight columns exactly zero, and the criterion on every
    tensor."""
    want = tuple(w for w in want if w != "h0" or h0 != "none")
    m = mirror(plan, n_ops, cin, B)
    fwd_ok, bwd_ok = _check_support(plan, n_ops, cin)
    assert fwd_ok and bwd_ok, what
    x, H0, wcat, bcat, wgt = _inputs(plan, n_ops, cin, B, T, seed, h0, bias)
    img = ops.gru_weight_image(wcat, bcat) if wimage else None
    with torch.no_grad(), _counted() as c:
        inf = ops.gru_seq_fwd(plan, n_ops, x, wcat, bcat, h0=H0, wimage=img)
    _assert_launches(c, _expect(m), what)
    LAUNCHED.add(("fwd", m[1], cin, n_ops))
    with _counted() as c:
        got = _fused(plan, n_ops, x, H0, wcat, bcat, wgt, want, bias, wimage)
    _assert_launches(c, _expect(m, bwd=bool(want), wgrad="w" in want), what)
    if want:
        LAUNCHED.add(("bwd", m[3], m[4], cin, n_ops))
    assert torch.equal(got[0], inf), (what, "training forward differs from inference")
    r64, r32 = _refs(plan, ops64, n_ops, x, H0, wcat, bcat, wgt, want, bias)
    if "w" in want:
        assert bool((got[3][~_live(n_ops, cin)] == 0).all()), (what, "dwcat outside the layout's columns")
    if plan.amplifying and n_ops:                 # see _op_scale: every step alone, and the backward kernels alone
        _one_steps(errs, plan, ops64, n_ops, x, H0, wcat, bcat, r64[0], m, what)
        if want:
            _stash_case(errs, plan, ops64, cin, B, T, seed, m, what + ("stash",), n_ops)
        return got
    _compare(errs, got, r32, r64, n_ops, m, what, T * B * plan.num_nodes, T)
    if T >= LONG_T and want:                       # the backward kernels alone, held to 4x (see _allow)
        _stash_case(errs, plan, ops64, cin, B, T, seed, m, what + ("stash",), n_ops)
    return got


# L = D - A scaled with a lambda_max below its default, 2 max(degree), leaves a spectrum beyond [-1, 1]: Chebyshev K = 2, lambda_max =
# 1.7 on 207-node hubs scales the hub's diagonal to 145.  The step's pre-activations are then sums of operands up to 145 times the state, and the recurrence
# multiplies rounding: with T = 9 a perturbation of H0 grew up to 7e5-fold in float64, and the fused output's error from float64 was 26x
# the op-for-op path's (0.16 against 0.006), so comparing whole windows measures the amplification (on the 129-node random and
# 206-node mod4 graphs, whose entries stay below 10, windows still reached 6.6x on the output and 7.5x on dH0).  Taken step by step from the float64
# state, the fused step's error was 0.5x to 5.2x the fp32 step's (up to 13.6x in single-window cases, where a maximum over fewer values
# leaves e32 small by chance), and of the same order as an exact emulation of the kernel's operands -- each fp32 operand split into fp16
# hi and lo (22 bits, where fp32 keeps 24), products exact, sums in float64 -- whose error was 0.1x to 2.2x the fused step's.  So the
# loss is the hi / lo split of the tensor-core operands (dcrnn_seq_tc.cu), inherent to the design and relative to the operands, not a
# defect.  Such a case (`plan.amplifying`, set by `build`) is held, instead, to: every step from the float64 state within 4x the fp32 step plus 2^-20 of
# the operands' scale, the largest entry times the state's (`_one_steps`: a cancelling sum scaled by its largest terms, as earlier files
# accept), and the backward kernels on the float64 stash within 4x (`_stash_case`).
def _op_scale(ops64, n_ops):
    """Largest magnitude of an entry of the operators the call uses (1 when it uses none)."""
    return max([1.0] + [float(ops64[k].abs().max()) for k in range(n_ops)])


def _one_steps(errs, plan, ops64, n_ops, x, H0, wcat, bcat, out64, m, what):
    """Every step of the window alone: the fused step from the float64 state rounded to fp32, against float64 from that state."""
    for t in range(x.size(1)):
        h = H0 if t == 0 else out64[:, t - 1].float().contiguous()
        xt = x[:, t:t + 1].contiguous()
        with torch.no_grad():
            with _counted() as c:
                got = ops.gru_seq_fwd(plan, n_ops, xt, wcat, bcat, h0=h)
            _assert_launches(c, _expect(m), what + (t,))
            r32 = _restated(plan, n_ops, xt, h, wcat, bcat)
            with _float64():
                r64 = _restated(None, n_ops, xt.double(), None if h is None else h.double(), wcat.double(), bcat.double(),
                                spmm=lambda k, u: ops64[k] @ u)
        scale = _op_scale(ops64, n_ops) * max(1.0, float(r64.abs().max()), 0.0 if h is None else float(h.abs().max()))
        _check_err(errs, FAM + "forward, one step from the float64 state", got, r32, r64, what + ("step", t), scale=scale)


# Departures from 4x, measured on an H100 (80 GB HBM3, 700 W) in the first run of this file:
#  * gradients through T >= 40 steps: dconv2, N = 16 hubs, cin 4, no bias, B = 3, T = 40 reached 4.7x the op-for-op path's error (1.19
#    of the 4x allowance).  `_run` also feeds the backward kernels the float64 stash of every such case and holds them to 4x, so the loss
#    is the forward's stash error carried back through 40 steps -- the reason test_gpu_dcrnn_narrow_envelope.py allows its K = 4
#    gradients 8x.  Allowed 8x.
#  * weight gradients contracted over more than 65 536 rows: at B = 2 SMs + 5, T = 2, N = 207 (111 366 rows) dwcat reached 11.7x the
#    op-for-op error (1.66 of the allowance; n_ops 1, cin 1; up to 1.44 at the other cin and n_ops).  The tensor cores' fp32
#    accumulation truncates (wgrad_tc.cu) along a chain of about rows / (16 SMs) tiles per partial, where the op-for-op path's cuBLAS
#    products sum 55 683 rows per step; every entry is a cancelling sum over all rows, scaled by the largest.  Allowed 16x.  The
#    contraction alone (test_wgrad_contraction_vs_float64) stays within 4x up to 12 * 5 * 207 rows and reaches 7.8x (1.14 of the
#    allowance) at those 111 366 rows: most of the departure is the contraction's own.
LONG_T, LONG_ROWS = 40, 65536


def _allow(i, rows, T):
    if i >= 3 and rows > LONG_ROWS:
        return 16
    return 8 if i >= 1 and T >= LONG_T else 4


def _compare(errs, got, r32, r64, n_ops, m, what, rows, T):
    for i, name in enumerate(("out", "dX", "dH0", "dwcat", "dbcat")):
        assert (got[i] is None) == (r64[i] is None), (what, name, "gradient returned / missing")
        if r64[i] is not None:
            fam = f"forward n_ops {n_ops}" if i == 0 else f"backward {m[3]} {m[4]}"
            _check_err(errs, FAM + fam, got[i], r32[i], r64[i], what + (name,), _allow(i, rows, T))


def _steps(cin, j):
    """T cycles through 1, 2, either side of T cin = 8 and 32 (the workspace pitch and the prologue's gather pass), and 40 steps."""
    ts = sorted({1, 2, 8 // cin - 1, 8 // cin, 8 // cin + 1, 32 // cin - 1, 32 // cin + 1, 40} - {0})
    return ts[j % len(ts)]


# ==== 1. the plan operators are the oracle's, rounded ===================================================================================
@pytest.mark.parametrize("name,flavor,n_ops,kw", PLANS, ids=[p[0] for p in PLANS])
def test_plan_operators_are_the_oracle_rounded(name, flavor, n_ops, kw):
    for n, kind in GEOS:
        if kind == "dups" and flavor != "dconv":
            kind = "random"
        if n == 1 and kw.get("norm", "sym") is None and kw.get("lam") is None:
            continue                                     # L = D - A = 0 and lambda_max = 2 max(w) = 0: 0 / 0 in both
        plan, ops64 = build(flavor, _graph(kind, n), n, **kw)
        for op, A64 in enumerate(ops64):
            A = _plan_dense(plan, op)
            want = A64.float().double()
            # a few ulps, and the plan's fp32 sums of the degrees: under L = D - A with a given lambda_max the hubs' diagonal (206
            # edges) came 8.6e-7 (6.5e-7 of the entry) from the rounded oracle; an operator in the wrong order or meaning is off by O(1e-2)
            tol = 2.0 ** -21 * float(want.abs().max()) + 2.0 ** -19 * want.abs()
            bad = (A - want).abs() > tol
            assert not bool(bad.any()), (name, n, kind, op, float((A - want).abs().max()), int(bad.sum()))


# ==== 2. plans x cin x bias across node counts, graph kinds and step counts =============================================================
@pytest.mark.parametrize("name,flavor,n_ops,kw", PLANS, ids=[p[0] for p in PLANS])
def test_plans_channels_and_bias_vs_float64(name, flavor, n_ops, kw):
    errs = []
    s = PLANS.index((name, flavor, n_ops, kw))
    for j, (cin, bias) in enumerate(itertools.product((1, 2, 3, 4), (True, False))):
        n, kind = GEOS[(5 * s + j) % len(GEOS)]
        if kind == "dups" and flavor != "dconv":
            kind = "random"
        if n == 1 and kw.get("norm", "sym") is None and kw.get("lam") is None:
            n, kind = 2, "random"
        plan, ops64 = build(flavor, _graph(kind, n), n, **kw)
        B, T = 1 + (j + s) % 3, _steps(cin, j + s)
        _run(errs, plan, ops64, n_ops, cin, B, T, 1000 * s + j, (name, n, kind, cin, bias, B, T), bias=bias, wimage=bool(j % 2))
    assert not errs, errs[:6]


@pytest.mark.parametrize("lam", [None, 1.7])
def test_unnormalized_laplacian_on_hubs_vs_float64(lam):
    """Chebyshev K = 2 with L = D - A on 207-node hubs, T = 9: at the default lambda_max (2 max(degree)) the operator's entries stay
    within 1 and the whole window is held to 4x; at 1.7 they reach 145 and each step is held alone (see `_op_scale`)."""
    plan, ops64 = build("cheb", _graph("hubs", 207), 207, norm=None, lam=lam)
    assert plan.amplifying == (lam is not None) and (_op_scale(ops64, 1) > 100) == (lam is not None) and _op_scale(ops64, 1) < 1.01 + 200 * (lam is not None)
    errs = []
    for cin in (1, 2, 3, 4):
        _run(errs, plan, ops64, 1, cin, 3, 9, cin, ("None", lam, cin))
    assert not errs, errs[:6]


# ==== 3. every launch variant: windows across SMs / 2 and SMs, staged and global graphs =================================================
def _variant_plan(n_ops, kind="hubs", n=207, edges=None):
    g = make_sized_graph("edges", n, edges) if edges else _graph(kind, n)
    if n_ops == 2:
        return build("dconv", g, n)
    return build("cheb", g, n, norm="sym")


def _staged_limit(n, cin, n_ops):
    """Largest edge count per operator whose transposed operators the backward still stages (graph_in_smem)."""
    e = 0
    while bwd_staged(n, cin, [e + 1] * n_ops):
        e += 1
    return e


@pytest.mark.parametrize("cin", [1, 2, 3, 4])
@pytest.mark.parametrize("n_ops", [0, 1, 2])
def test_windows_and_launch_variants_vs_float64(n_ops, cin):
    """B = 1, 2, 3, SMs / 2, SMs / 2 + 1, SMs, SMs + 1 and 2 SMs + 5 at N = 207: forward CTA pair, one CTA, one persistent CTA per SM;
    backward CTA pair and one CTA.  At two operators also a graph one edge past the backward's staged-copy limit (global CSR)."""
    S = _sms()
    errs = []
    plan, ops64 = _variant_plan(n_ops)
    for j, B in enumerate((1, 2, 3, S // 2, S // 2 + 1, S, S + 1, 2 * S + 5)):
        _run(errs, plan, ops64, n_ops, cin, B, 2 if B > 3 else 3, 10 * cin + j, ("hubs", 207, n_ops, cin, B), wimage=bool(j % 2))
    if n_ops == 2:
        e = _staged_limit(207, cin, 2) + 1
        plan, ops64 = _variant_plan(2, edges=e)
        assert mirror(plan, 2, cin, 1)[4] == "global"
        for B in (1, S // 2 + 1):
            _run(errs, plan, ops64, n_ops, cin, B, 3, 7 * cin + B, ("edges", 207, e, n_ops, cin, B))
    assert not errs, errs[:6]


def test_one_operator_densest_image_and_staged_limit():
    """At one operator the densest graph that still has both images (forward + training, the backward stages it), one edge more (no
    image: gru_seq_supported is false), and the staged-copy limit of each cin, whose far side only the stash path below reaches."""
    e = 0
    while image_fits(207, 1, e + 1):
        e += 1
    plan, _ = build("dconv", make_sized_graph("edges", 207, e + 1), 207)
    assert not ops.gru_seq_supported(plan, 1, 2, 32) and not mirror(plan, 1, 2, 1)[0]
    plan, ops64 = build("dconv", make_sized_graph("edges", 207, e), 207)
    errs = []
    for cin in (1, 2, 3, 4):
        assert mirror(plan, 1, cin, 1)[4] == "staged"
        _run(errs, plan, ops64, 1, cin, 2, 3, cin, ("densest", e, cin))
    assert not errs, errs[:6]


def test_one_operator_global_csr_backward_from_a_float64_stash():
    """The backward's global-CSR variant at n_ops = 1 is unreachable through ops.gru_seq_train: the forward needs a graph image, which
    holds fewer entries at any N <= 207 than the backward's staged copy does at N = 207 (where the staged copy is smallest; the basis
    is 72 columns for every cin at one operator).  Both numbers are computed here.  So the backward kernels run on the float64 forward's
    output and stash rounded to fp32, for each cin on both sides of the staged-copy limit, CTA pair and one CTA."""
    image_max = 0
    while image_fits(1, 1, image_max + 1):
        image_max += 1
    limits = {cin: _staged_limit(207, cin, 1) for cin in (1, 2, 3, 4)}
    assert image_max < min(limits.values()), (image_max, limits)
    errs = []
    S = _sms()
    for cin, lim in limits.items():
        for e in (lim, lim + 1):
            plan, ops64 = build("dconv", make_sized_graph("edges", 207, e), 207)
            fwd_ok, bwd_ok = _check_support(plan, 1, cin)
            assert bwd_ok and not fwd_ok
            for B in (1, S // 2 + 1):
                m = mirror(plan, 1, cin, B)
                assert m[4] == ("staged" if e == lim else "global")
                _stash_case(errs, plan, ops64, cin, B, 2, 100 * cin + B, m, ("stash", e, cin, B))
    assert not errs, errs[:6]


def _stash_case(errs, plan, ops64, cin, B, T, seed, m, what, n_ops=1):
    x, H0, wcat, bcat, wgt = _inputs(plan, n_ops, cin, B, T, seed, "window", True)
    want = ("x", "h0", "w")
    lv = _leaves(lambda t: t.detach().double(), x, H0, wcat, bcat, want, True)
    stash64 = []
    with _float64():
        out64 = _restated(None, n_ops, *lv, spmm=lambda k, t: ops64[k] @ t, stash=stash64)
    g64 = _loss_grads([out64], [wgt.double()], lv)
    l32 = _leaves(lambda t: t.detach().clone(), x, H0, wcat, bcat, want, True)
    g32 = _loss_grads([_restated(plan, n_ops, *l32)], [wgt], l32)
    out = out64.detach().float()
    stash = torch.stack([torch.stack(s, 1) for s in stash64], 1).detach().float().contiguous()     # (B, T, 3, N, 32)
    N = plan.num_nodes
    f32 = dict(device=DEV, dtype=torch.float32)
    ld = ops.gru_bwd_basis_ld(n_ops, cin)
    S1, S2 = torch.empty(T * B, N, ld, **f32), torch.empty(T * B, N, ld, **f32)
    dph, dpzr = torch.empty(T, B, N, 32, **f32), torch.empty(T, B, N, 64, **f32)
    dX, dH0 = torch.empty(B, T, N, cin, **f32), torch.empty(B, N, 32, **f32)
    gout = wgt / wgt.numel()
    with _counted() as c:
        whsT, wzrT = ops.gru_pack_bwd_weights(n_ops, cin, wcat)
        ops.gru_bwd_basis(plan, n_ops, x, out, H0, stash, S1, S2)
        ops.gru_bwd_seq(plan, n_ops, cin, gout, out, H0, stash, whsT, wzrT, dph, dpzr, dX, dH0)
        dW, dB = ops.gru_bwd_wgrad(n_ops, cin, S1, S2, dpzr, dph, True)
    _assert_launches(c, _expect(m, fwd=False, bwd=True, wgrad=True), what)
    LAUNCHED.add(("bwd", m[3], m[4], cin, n_ops))
    for name, got, r32, r64 in zip(("dX", "dH0", "dwcat", "dbcat"), (dX, dH0, dW, dB), g32, g64):
        _check_err(errs, FAM + f"backward on the float64 stash {m[3]} {m[4]}", got, r32, r64, what + (name,))


def test_65536_windows_forward_on_a_sample_vs_float64():
    """What the TGCN fall-back sends for more than 65 535 batch rows: 65 536 one-step windows, persistent over the SMs."""
    S = _sms()
    plan, ops64 = build("gcn", _graph("mod4", 16), 16)
    B, cin = 65536, 2
    x, H0, wcat, bcat, _ = _inputs(plan, 1, cin, B, 1, 3, "window", True)
    m = mirror(plan, 1, cin, B)
    assert m[1] == "persistent"
    with torch.no_grad(), _counted() as c:
        out = ops.gru_seq_fwd(plan, 1, x, wcat, bcat, h0=H0)
    _assert_launches(c, _expect(m), "65536 windows")
    LAUNCHED.add(("fwd", m[1], cin, 1))
    pick = sorted({0, 1, S - 1, S, S + 1, 2 * S, B // 2, B - S - 1, B - 1} | set(range(7, B, 4099)))
    with torch.no_grad():
        with _float64():
            r64 = _restated(None, 1, x[pick].double(), H0[pick].double(), wcat.double(), bcat.double(), spmm=lambda k, t: ops64[k] @ t)
        r32 = _restated(plan, 1, x[pick], H0[pick], wcat, bcat)
    errs = []
    _check_err(errs, FAM + "forward n_ops 1", out[pick], r32, r64, ("65536 windows",))
    assert not errs, errs


def test_node_limit_208_routes_elsewhere():
    """N = 208 is past the 8-bit graph images: gru_seq_supported is false for every operator count, gru_bwd_supported is what
    fits_one_sm says, and GConvGRU takes the row-split cell."""
    g = make_graph("random", 208)
    plan, _ = build("cheb", g, 208, norm="sym")
    for n_ops in (0, 1):
        for cin in (1, 4):
            assert not ops.gru_seq_supported(plan, n_ops, cin, 32)
            assert ops.gru_bwd_supported(plan, n_ops, cin, 32) == _fits_one_sm(208, cin, n_ops) == mirror(plan, n_ops, cin, 1)[2]
    ei = torch.from_numpy(np.stack(g[:2])).to(DEV)
    ew = torch.from_numpy(g[2]).to(DEV)
    for K in (1, 2):
        torch.manual_seed(K)
        m = GConvGRU(2, 32, K).to(DEV)
        X, H = torch.randn(208, 2, device=DEV), 0.5 * torch.randn(208, 32, device=DEV)
        with torch.no_grad(), _counted() as c:
            out = m(X, ei, ew, H)
        assert not [k for k in c if k.startswith(("k_dcrnn_seq", "k_gru_bwd"))] and c.get("k_gru_rows_fwd_a"), (K, c)
        with _float64():
            p64 = {k: v.double() for k, v in m.state_dict().items()}
            ref = R.gconv_gru_cell(p64, X.double(), ei, ew.double(), H.double())
        assert torch.allclose(out.double(), ref, rtol=1e-4, atol=1e-5), (K, float((out.double() - ref).abs().max()))
        with _counted() as c:
            m(X.requires_grad_(True), ei, ew, H).square().mean().backward()
        assert not [k for k in c if k.startswith(("k_dcrnn_seq", "k_gru_bwd"))], (K, c)


# ==== 4. states, gradient subsets and weight images =====================================================================================
@pytest.mark.parametrize("n_ops", [0, 1, 2])
def test_states_and_gradient_subsets_vs_float64(n_ops):
    """h0 absent or per window, every subset of {X, h0, parameters} requiring grad (none: the forward alone), with and without the
    weight image; then a shared h0 of shape (N, 32) and (1, N, 32) in the forward, and the backward's refusal of a shared h0."""
    n, kind = (129, "sink") if n_ops == 2 else (65, "mod4")
    plan, ops64 = build("dconv", _graph(kind, n), n) if n_ops == 2 else build("cheb", _graph(kind, n), n, norm="sym")
    errs = []
    j = 0
    for h0 in ("none", "window"):
        grads = ("x", "w") if h0 == "none" else ("x", "h0", "w")
        for k in range(len(grads) + 1):
            for want in itertools.combinations(grads, k):
                cin = 1 + j % 4
                _run(errs, plan, ops64, n_ops, cin, 3, 4, 50 + j, (h0, want, cin), h0=h0, want=want, wimage=bool(j % 2))
                j += 1
    cin, B, T = 3, 4, 3
    x, _, wcat, bcat, _ = _inputs(plan, n_ops, cin, B, T, 77, "none", True)
    Hs = 0.5 * torch.randn(n, 32, device=DEV)
    with _float64():
        r64 = _restated(None, n_ops, x.double(), Hs.double(), wcat.double(), bcat.double(), spmm=lambda k, t: ops64[k] @ t)
    with torch.no_grad():
        r32 = _restated(plan, n_ops, x, Hs, wcat, bcat)
    m = mirror(plan, n_ops, cin, B)
    for shape in ((n, 32), (1, n, 32)):
        with torch.no_grad(), _counted() as c:
            out = ops.gru_seq_fwd(plan, n_ops, x, wcat, bcat, h0=Hs.reshape(shape), h0_shared=True)
        _assert_launches(c, _expect(m), ("shared h0", shape))
        _check_err(errs, FAM + f"forward n_ops {n_ops}", out, r32, r64, ("shared h0", shape))
        assert torch.equal(out, ops.gru_seq_fwd(plan, n_ops, x, wcat, bcat, h0=Hs.expand(B, n, 32).contiguous()))
    assert not errs, errs[:6]
    # the backward serves a dense (B, N, 32) h0 only
    L, p = _lib.lib(), _lib.ptr
    f = torch.zeros(1 << 20, device=DEV)
    n0 = _lib.launch_count()
    for rc in (L.stmp_gru_bwd_seq(plan.handle, n_ops, B, T, cin, p(f), p(f), p(f), 0, p(f), p(f), p(f), p(f), p(f), None, p(f), None),
               L.stmp_gru_bwd_basis(plan.handle, n_ops, B, T, cin, p(f), T * n * cin, n * cin, p(f), p(f), 0, p(f), p(f), p(f),
                                    ops.gru_bwd_basis_ld(n_ops, cin), None)):
        with pytest.raises(_lib.StmpUnsupported, match="shared h0"):
            _lib.check(rc)
    assert _lib.launch_count() == n0


def test_state_size_guards_raise_before_any_launch():
    """ops.gru_seq_fwd reads h0 at a batch stride of N * 32 (0 when shared) and ops.dcrnn_seq_fwd at N * cout: an h0 that holds
    another count would be read past its end or silently start every window from state 0."""
    n, B, cin = 20, 3, 2
    g = _graph("random", n)
    plan, _ = build("cheb", g, n, norm="sym")
    dplan, _ = build("dconv", g, n)
    x, H0, wcat, bcat, _ = _inputs(plan, 1, cin, B, 2, 5, "window", True)
    torch.manual_seed(0)
    dm = BatchedDCRNN(cin, 32, 2).to(DEV)
    calls = {
        "per-window (N, 32)": lambda: ops.gru_seq_fwd(plan, 1, x, wcat, bcat, h0=H0[0]),
        "per-window (1, N, 32)": lambda: ops.gru_seq_fwd(plan, 1, x, wcat, bcat, h0=H0[:1]),
        "per-window (B - 1, N, 32)": lambda: ops.gru_seq_fwd(plan, 1, x, wcat, bcat, h0=H0[:2]),
        "shared (B, N, 32)": lambda: ops.gru_seq_fwd(plan, 1, x, wcat, bcat, h0=H0, h0_shared=True),
        "training (N, 32)": lambda: ops.gru_seq_train(plan, 1, x, H0[0], wcat, bcat, None, [("w", 0, 96, 0, 112)],
                                                      [wcat.clone().requires_grad_(True)]),
        "dcrnn (N, 32)": lambda: ops.dcrnn_seq_fwd(dplan, x, *dm._params(), 2, h0=H0[0]),
        "dcrnn (1, N, 32)": lambda: ops.dcrnn_seq_fwd(dplan, x, *dm._params(), 2, h0=H0[:1]),
    }
    for what, call in calls.items():
        n0 = _lib.launch_count()
        with pytest.raises(RuntimeError, match="elements, the kernel indexes"):
            call()
        assert _lib.launch_count() == n0, what
    with torch.no_grad():                                 # the sizes the kernels index are accepted
        ops.gru_seq_fwd(plan, 1, x[:1], wcat, bcat, h0=H0[0])
        ops.gru_seq_fwd(plan, 1, x, wcat, bcat, h0=H0[0], h0_shared=True)
        ops.dcrnn_seq_fwd(dplan, x[:1], *dm._params(), 2, h0=H0[0])


# ==== 5. determinism: CTA pair = one CTA, repeats bit-identical ==========================================================================
@pytest.mark.parametrize("n_ops", [0, 1, 2])
def test_pair_equals_one_cta_and_repeats_are_bit_identical(n_ops):
    for n, kind in ((16, "hubs"), (129, "random"), (207, "mod4")):
        plan, _ = _variant_plan(n_ops, kind, n)
        cin = 1 + (n + n_ops) % 4
        x, H0, wcat, bcat, wgt = _inputs(plan, n_ops, cin, 2, 3, n, "window", True)
        want = ("x", "h0", "w")
        runs = []
        for split in (1, 1, 0):
            with _option("dcrnn_fwd_split", split, 1), _option("dcrnn_bwd_split", split, 1), _counted() as c:
                runs.append(_fused(plan, n_ops, x, H0, wcat, bcat, wgt, want, True))
            m = mirror(plan, n_ops, cin, 2, fwd_split=bool(split), bwd_split=bool(split))
            _assert_launches(c, _expect(m, bwd=True, wgrad=True), (n, split))
            LAUNCHED.add(("fwd", m[1], cin, n_ops))
            LAUNCHED.add(("bwd", m[3], m[4], cin, n_ops))
        for a, b, d in zip(*runs):
            assert torch.equal(a, b), (n, "repeat differs")
            assert torch.equal(a, d), (n, "CTA pair differs from one CTA", float((a - d).abs().max()))


# ==== 6. the module ======================================================================================================================
@pytest.mark.parametrize("norm", ["sym", "rw", None])
@pytest.mark.parametrize("K", [1, 2])
def test_gconv_gru_module_vs_float64(K, norm):
    """GConvGRU over bias x {H None, a leaf H, H carried for 5 steps} x {X requires grad or not}, fused against float64 (the oracle's
    cell) and the op-for-op path (`fused_training = False`)."""
    n = 129
    g = _graph("hubs", n)
    ei, ew = torch.from_numpy(np.stack(g[:2])).to(DEV), torch.from_numpy(g[2]).to(DEV)
    lam = 1.7 if norm == "rw" else None
    errs = []
    for j, (bias, hmode, xgrad) in enumerate(itertools.product((True, False), ("none", "leaf", "carried"), (False, True))):
        cin = 1 + (j + K) % 4
        torch.manual_seed(100 * K + j)
        m = GConvGRU(cin, 32, K, normalization=norm, bias=bias).to(DEV)
        with torch.no_grad():
            for name, p in m.named_parameters():
                if name.endswith("bias"):
                    p.normal_(0, 0.1)
        steps = 5 if hmode == "carried" else 1
        Xs = [torch.randn(n, cin, device=DEV) for _ in range(steps)]
        H0 = 0.5 * torch.randn(n, 32, device=DEV)
        wgts = [torch.randn(n, 32, device=DEV) for _ in range(steps)]
        names = [k for k, _ in m.named_parameters()]

        def run(fn, cast, params):
            xs = [cast(X).requires_grad_(xgrad) for X in Xs]
            h0 = None if hmode == "none" else cast(H0).requires_grad_(True)
            h, outs = h0, []
            for X in xs:
                h = fn(X, h)
                outs.append(h)
            leaves = xs + [h0] + params
            grads = _loss_grads(outs, [cast(w) for w in wgts], leaves)
            dX = torch.stack(grads[:steps]) if xgrad else None
            return [torch.stack([o.detach() for o in outs]), dX, grads[steps]] + grads[steps + 1:]

        p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
        lam64 = None if lam is None else torch.tensor(lam, dtype=torch.float64, device=DEV)
        with _float64():
            zeros64 = torch.zeros(n, 32, dtype=torch.float64, device=DEV)
            r64 = run(lambda X, h: R.gconv_gru_cell(p64, X, ei, ew.double(), zeros64 if h is None else h, lambda_max=lam64,
                                                   normalization=norm), lambda t: t.detach().double(), [p64[k] for k in names])
        params = list(m.parameters())
        res = {}
        for fused in (False, True):
            m.fused_training = fused
            m.zero_grad(set_to_none=True)
            with _counted() as c:
                res[fused] = run(lambda X, h: m(X, ei, ew, h, lambda_max=lam), lambda t: t.detach().clone(), params)
        want = {"k_dcrnn_seq_tc": steps, "k_gru_bwd_seq": steps, "k_gru_pack_bwd_weights": steps}
        assert {k: c.get(k, 0) for k in want} == want and "k_spmm" not in c, (K, norm, j, c)
        what = (K, norm, bias, hmode, xgrad, cin)
        for name, got, r32, rr in zip(["out", "dX", "dH0"] + names, res[True], res[False], r64):
            assert (got is None) == (rr is None), (what, name)
            if rr is not None:
                _check_err(errs, FAM + "GConvGRU module", got, r32, rr, what + (name,))
    assert not errs, errs[:6]


# ==== 7. the weight-gradient contraction on its own ======================================================================================
@pytest.mark.parametrize("cin", [1, 2, 3, 4])
@pytest.mark.parametrize("n_ops", [0, 1, 2])
def test_wgrad_contraction_vs_float64(n_ops, cin):
    """stmp_gru_bwd_wgrad at (n_ops + 1)(cin + 32) = 33 .. 108 columns: 1, 15, 16 and 17 rows, fewer 16-row tiles than SMs, more tiles
    than partials, 12 * 5 * 207 and 111 366 rows (past `LONG_ROWS`); d pre-activations at mean-loss magnitudes (1e-6 .. 1e-10), which the TF32 hi / lo split must not
    flush; the basis's padding columns hold NaN and must not reach a result; dwcat is zero wherever the layout has no column."""
    S = _sms()
    ld, C = ops.gru_bwd_basis_ld(n_ops, cin), cin + 32
    C3 = (n_ops + 1) * C
    cols = torch.tensor([96 + 4 * b + c if c < cin else 32 * b + c - cin for b in range(n_ops + 1) for c in range(C)], device=DEV)
    live = _live(n_ops, cin)
    errs = []
    gen = torch.Generator(device=DEV).manual_seed(n_ops * 4 + cin)
    for rows in (1, 15, 16, 17, 16 * (S - 5) + 3, 16 * (S + 7) + 5, 12 * 5 * 207, 2 * 269 * 207):
        for mag in (1e-6, 1e-10):
            S1 = torch.randn(rows, 1, ld, device=DEV, generator=gen)
            S2 = torch.randn(rows, 1, ld, device=DEV, generator=gen)
            S1[..., C3:] = float("nan")
            S2[..., C3:] = float("nan")
            dpzr = torch.randn(rows, 64, device=DEV, generator=gen) * mag
            dph = torch.randn(rows, 32, device=DEV, generator=gen) * mag
            with _counted() as c:
                dW, dB = ops.gru_bwd_wgrad(n_ops, cin, S1, S2, dpzr, dph, True)
            _assert_launches(c, {"k_dcrnn_wgrad_tc": 1, "k_gru_wgrad_reduce": 1}, rows)
            refs = []
            for cast in (lambda t: t.double(), lambda t: t):
                a1, a2 = cast(S1[:, 0, :C3]), cast(S2[:, 0, :C3])
                W = torch.zeros(96, 112, dtype=a1.dtype, device=DEV)
                W[:64, cols] = (a1.t() @ cast(dpzr)).t()
                W[64:, cols] = (a2.t() @ cast(dph)).t()
                refs.append((W, torch.cat([cast(dpzr).sum(0), cast(dph).sum(0)])))
            (W64, b64), (W32, b32) = refs
            what = (n_ops, cin, rows, mag)
            assert bool((dW[~live] == 0).all()), (what, "dwcat outside the layout's columns")
            allow = _allow(3, rows, 1)                # beyond LONG_ROWS rows the departure of `_allow`, measured here on its own
            _check_err(errs, FAM + "wgrad", dW, W32, W64, what + ("dwcat",), allow)
            _check_err(errs, FAM + "wgrad", dB, b32, b64, what + ("dbcat",), allow)
    assert not errs, errs[:6]
