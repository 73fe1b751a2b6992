"""DyGrEncoder on the H100: the gated plan bit-exact against a CPU restatement, every golden case fused and op for op against the float64
oracle (held to the reference's fingerprints by tests/test_dygrae_cpu.py), the envelope against float64, bit-equal training and inference
forwards, repeatable and loss-scale-equivariant gradients, exact launch counts, the layer limit, the weight-gradient reduce bit for bit,
the routes outside the envelope, CUDA-graph replay and the ABI's errors.

Envelope criterion (test_gpu_rows_envelope.py's): dygrae_step in float64 on the GPU with autograd is the reference, dygrae_step in float32
(no TF32) the yardstick -- with the module's own cuDNN LSTM as its LSTM stage wherever the module uses cuDNN (_yardstick); every tensor --
H_tilde, H, C, dX when wanted, dH and dC when H and C are given, each parameter's gradient on its own -- stays within 4x the yardstick's
error plus 2^-20 of its scale (at C <= 2 the parameter gradients share the model's largest as their scale, and cases behind the cuDNN
LSTM are allowed 8x: _dy_case says why).  Every case asserts the launches (_dy_launches).  Shapes: C 1, 2, 15, 16, 17, 31, 32 with cin 1, C - 1, C (C 16 | 17: the row-split LSTM cell |
cuDNN); L_g 1, 2, 3, 8, 33, and 1 024 for inference (deep stacks contracted, _contract); N 1, 2, 15, 16, 17, 31, 32, 33, 4 224, 4 225 and
50 000 (the weight gradient's 32-row tiles span two layers when N % 32 != 0); rings, every in- and out-degree residue mod 4, hubs,
duplicates, self loops, rows without in-edges, E = 0; edge weights None, positive and signed with exact zeros; H and C None or given; a
5-step carried sequence.

max is compared only where float32 and float64 take the same argmax: at L_g = 1 on dyadic inputs whose every message is exact in both
(exact ties of duplicated edges and of distinct sources, maxima of exactly +0 and -0.0, empty rows, in-degree 1..9; 70 and 50 000 nodes),
and at L_g >= 2 on seeded random inputs whose float64 forward keeps every top-two gap of a row and channel at least 2^-16 of its layer's
largest message, which the test asserts before comparing.

Largest ratios of one run on an H100 80GB HBM3 at a 700 W power limit, as printed by `_report`:
    ggc_rows add    e / e32 5.93   used 0.88
    ggc_rows mean   e / e32 3.88   used 0.52
    ggc_rows max    e / e32 4.17   used 0.76
This file and test_gpu_lrgcn.py took 121 s together there.
"""
import contextlib
import ctypes
import os

import numpy as np
import pytest
import torch

from dygrae_seq import aggregate, dygrae_step, ggc, gru_cell, load, model_for, oracle_run, run, states_for
from gconvgru_seq import chickenpox_train_split
from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.nn.recurrent import DyGrEncoder
from pytorch_geometric_temporal_b200.plan import GatedPlan, GraphPlan
from test_gpu_lrgcn import _Relation
from test_gpu_rows_envelope import WORST, _check_err, _counted, _float64, _loss_grads, _or_zeros, check_family, make_graph
from test_gpu_wgrad_reduce import _ar, _check, _equal, _parts, _randn, _rows, _sms, _sum, _workspace, NAN
from wikimaths_seq import load as load_wikimaths

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
AGGRS = ("add", "mean", "max")


@pytest.fixture(autouse=True)
def _cudnn_fp32():
    """cuDNN's LSTM (the C > 16 and two-layer routes), the op-for-op path and the fp32 yardstick in full fp32: by default torch lets
    cuDNN round operands to TF32, about 1e-3 off the float64 oracle; cuBLAS's TF32 switch is turned off too."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _plan_cpu(ei, ew, n, aggr):
    """(rowptr, col, val, eid) by destination and by source: every edge in edge order, val = w (add, max) or w / cnt(dst) (mean)."""
    src, dst = ei[0], ei[1]
    w = torch.ones(ei.size(1)) if ew is None else ew.float()
    if aggr == "mean":
        w = w / torch.bincount(dst, minlength=n).float()[dst]
    out = []
    for key, other in ((dst, src), (src, dst)):
        order = torch.sort(key, stable=True).indices
        rowptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(torch.bincount(key, minlength=n), 0)])
        out.append((rowptr.int(), other[order].int(), w[order].float(), order.int()))
    return out


def _graph_of(kind, n, seed):
    """edge_index of a named geometry on n nodes."""
    g = torch.Generator().manual_seed(seed)
    if kind == "empty":
        return torch.zeros(2, 0, dtype=torch.int64)
    if kind == "one_node":
        return torch.tensor([[0, 0], [0, 0]])                                   # a duplicated self loop on the only node
    e = 4 * n
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, max(1, n - 3), (e,), generator=g)                    # the last nodes have no in-edge
    if kind == "hub":
        dst[:400] = 0                                                           # a 400-edge hub
        src[400:800] = 1                                                        # and a 400-edge source
    ei = torch.stack([src, dst])
    return torch.cat([ei, ei[:, :e // 8], torch.stack([src[:5], src[:5]])], 1)  # duplicates (exact max ties) and self loops


def _weights(kind, E, seed):
    if kind is None:
        return None
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(E, generator=g) * 2
    if kind == "signed":
        w = w - 1
        w[::7] = 0.0                                                            # zero and negative weights
    return w


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("n,kind,wk", [(20, "random", None), (300, "hub", "signed"), (7, "empty", None), (1, "one_node", "pos")])
def test_plan_bit_exact(aggr, n, kind, wk):
    ei = _graph_of(kind, n, n)
    ew = _weights(wk, ei.size(1), 3)
    plan = GatedPlan(ei.to(DEV), None if ew is None else ew.to(DEV), n, aggr)
    assert plan.n_ops == 1
    want = _plan_cpu(ei, ew, n, aggr)
    for t in (0, 1):
        got = [x.cpu() for x in plan.export(0, bool(t))]
        for a, b in zip(got, want[t]):
            assert torch.equal(a, b)


def test_plan_rejects_bad_graphs():
    ei = torch.tensor([[0, 5], [1, 0]], device=DEV)
    with pytest.raises(RuntimeError, match="outside"):
        GatedPlan(ei, None, 3, "add")
    out = ctypes.c_void_p()
    L = _lib.lib()
    assert L.stmp_plan_create_gated(3, 1, _lib.ptr(ei), None, 3, None, ctypes.byref(out)) == _lib.STMP_EINVAL
    assert L.stmp_plan_create(_lib.FLAVOR_GATED, 3, 1, _lib.ptr(ei), None, 0, -1.0, 0, None, ctypes.byref(out)) == _lib.STMP_EINVAL


def _graph(c):
    if c["graph"] == "chickenpox":
        return chickenpox_train_split()
    w = load_wikimaths(GOLDEN)
    return w["edge_index"], w["edge_weight"], w["X"], w["Y"]


def _close(got, want, what, rtol=2e-4):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = float(want.abs().max()) + 1e-30
    err = float((got - want).abs().max()) / scale
    assert err <= rtol, (what, err)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_golden_cases(name, fused):
    c = load(GOLDEN)["cases"][name]
    ei, ew, X, Y = _graph(c)
    H0, C0 = states_for(c, X.shape[1], dtype=torch.float64)
    outs64, cost64, leaves = oracle_run(c, X, Y, ei, ew, H0, C0)
    cost64.backward()
    m = model_for(c, DEV, fused)
    h0, c0 = states_for(c, X.shape[1], DEV)
    before = dict(_lib.path_counters())
    outs, cost = run(m, X.to(DEV), Y.to(DEV), ei.to(DEV), ew.to(DEV), h0, c0, c["state"] != "none")
    cost.backward()
    after = _lib.path_counters()
    ran = lambda k: after.get(k, 0) > before.get(k, 0)
    assert (ran("k_ggc_rows_fwd") or ran("k_ggc_rows_fwd_max")) is fused
    assert (ran("k_lstm_rows_fwd") or ran("k_lstm_wide_rows_fwd")) is (fused and c["C"] <= 16 and c["Ll"] == 1)
    assert abs(float(cost.detach()) - float(cost64.detach())) <= 1e-5 * abs(float(cost64.detach()))
    _close(outs, outs64, "out")
    for k, p in m.named_parameters():
        _close(p.grad, leaves[k].grad, k, 1e-3)
    if H0 is not None:
        _close(h0.grad, H0.grad, "gH0", 1e-3)
        _close(c0.grad, C0.grad, "gC0", 1e-3)


def _params64(m):
    return {k: v.detach().double().cpu().requires_grad_(True) for k, v in m.state_dict().items()}


def _check_step(m, c, X, ei, ew, H, C, want_dx, rtol=1e-3):
    """One fused step (conv route asserted) against dygrae_step in float64: outputs, every parameter's, X's, H's and C's gradient."""
    p64 = _params64(m)
    xs = [None if t is None else t.double().requires_grad_(want_dx or i > 0) for i, t in enumerate((X, H, C))]
    o64 = dygrae_step(p64, c, xs[0], ei, ew, xs[1], xs[2])
    g = torch.Generator().manual_seed(1)
    coef = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in o64]
    sum((a * b).sum() for a, b in zip(o64, coef)).backward()
    md = m.to(DEV)
    xd = [None if t is None else t.to(DEV).requires_grad_(want_dx or i > 0) for i, t in enumerate((X, H, C))]
    before = dict(_lib.path_counters())
    o = md(xd[0], ei.to(DEV), None if ew is None else ew.to(DEV), xd[1], xd[2])
    after = _lib.path_counters()
    assert sum(after.get(k, 0) - before.get(k, 0) for k in ("k_ggc_rows_fwd", "k_ggc_rows_fwd_max")) == c["Lg"]
    sum((a * b.float().to(DEV)).sum() for a, b in zip(o, coef)).backward()
    for a, b, what in zip(o, o64, ("H_tilde", "H", "C")):
        _close(a, b, what, 1e-4)
    for k, q in md.named_parameters():
        _close(q.grad, p64[k].grad, k, rtol)
    for t, ref, what in zip(xd, xs, ("dX", "dH", "dC")):
        if t is not None and t.requires_grad:
            _close(t.grad, ref.grad, what, rtol)


def _model(C, Lg, aggr, Ho, seed, Ll=1):
    torch.manual_seed(seed)
    m = DyGrEncoder(C, Lg, aggr, Ho, Ll)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.4)
    return m


# ---- the envelope against float64 (the criterion of test_gpu_rows_envelope.py) -------------------------------------------------------
FAMILIES = tuple(f"ggc_rows {a}" for a in AGGRS)
GGC = ("k_ggc_rows_msg", "k_ggc_rows_fwd", "k_ggc_rows_fwd_max", "k_ggc_rows_bwd", "k_ggc_rows_bwd_max", "k_ggc_rows_wgrad",
       "k_ggc_rows_wgrad_reduce")
CELL = ("k_lstm_rows_fwd", "k_lstm_rows_bwd_a", "k_lstm_rows_bwd_b", "k_dcrnn_wgrad", "k_lstm_rows_wgrad_reduce", "k_lstm_wide_rows_fwd",
        "k_lstm_wide_rows_bwd_a", "k_lstm_wide_rows_bwd_b", "k_lstm_wide_rows_wgrad", "k_lstm_wide_rows_wgrad_reduce")
OUTS = ("H_tilde", "H", "C")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for fam in FAMILIES:
        if fam in WORST:
            ratio, used, what = WORST[fam]
            print(f"\nDyGrEncoder envelope: {fam}: largest e / e32 = {ratio:.2f}, largest used fraction of the allowance = {used:.2f} at {what}")


def _ran(c):
    return {k: v for k, v in c.items() if k in GGC + CELL}


def _rows_lstm(c):
    return c["C"] <= 16 and c["Ll"] == 1


def _dy_launches(c, train, want_dx):
    """The row-split launches of one step (DESIGN §4r): forward L_g GatedGraphConv launches (one more for max's first messages) and the
    row-split LSTM cell when C <= 16 and L_l = 1; backward the LSTM cell's bwd_a and weight gradient, L_g GatedGraphConv backward launches
    plus one for dX (add, mean) or always (max), and the convolution's weight gradient and its reduce."""
    mx, L, wide = c["aggr"] == "max", c["Lg"], c["Ho"] == 64
    want = {"k_ggc_rows_msg": int(mx), "k_ggc_rows_fwd_max" if mx else "k_ggc_rows_fwd": L}
    if _rows_lstm(c):
        want["k_lstm_wide_rows_fwd" if wide else "k_lstm_rows_fwd"] = 1
    if train:
        want.update({"k_ggc_rows_bwd_max" if mx else "k_ggc_rows_bwd": L + int(mx or want_dx), "k_ggc_rows_wgrad": 1,
                     "k_ggc_rows_wgrad_reduce": 1})
        if _rows_lstm(c):
            want.update({"k_lstm_wide_rows_bwd_a": 1, "k_lstm_wide_rows_wgrad": 1, "k_lstm_wide_rows_wgrad_reduce": 1} if wide else
                        {"k_lstm_rows_bwd_a": 1, "k_dcrnn_wgrad": 1, "k_lstm_rows_wgrad_reduce": 1})
    return {k: v for k, v in want.items() if v}


def _yardstick(m, p, c, x, ei, ew, h, cc, cudnn=False):
    """dygrae_step from the parameter dict p, except that when the module hands the convolution's output to its cuDNN LSTM (C > 16, two
    LSTM layers, or `cudnn`: the op-for-op route) the LSTM stage is that same cuDNN LSTM on p's tensors: cuDNN's LSTM is up to ~30x further
    from float64 than the formula in float32, an error this project's kernels neither make nor can remove, so both sides carry it."""
    if _rows_lstm(c) and not cudnn:
        return dygrae_step(p, c, x, ei, ew, h, cc)
    Ht = ggc({k[len("conv_layer."):]: v for k, v in p.items() if k.startswith("conv_layer.")}, x, ei, ew, c["aggr"], c["C"])[None]
    lstm = {k[len("recurrent_layer."):]: v for k, v in p.items() if k.startswith("recurrent_layer.")}
    args = (Ht,) if h is None else (Ht, (h[None], cc[None]))
    out, (H, C) = torch.func.functional_call(m.recurrent_layer, lstm, args)
    return out.squeeze(), H.squeeze(), C.squeeze()


def _dy_case(errs, m, c, X, ei, ew, given, want_dx, seed, what, train=True):
    """One DyGrEncoder step on the row-split kernels against float64 (dygrae_step in float64, autograd), with _yardstick in float32 as
    the fp32 op-for-op error: H_tilde, H, C and, when `train`, dX (if wanted), dH and dC (if H and C are given) and every parameter's gradient.
    Asserts the launches of inference and training and that the training forward equals inference bit for bit.

    At C <= 2 a parameter gradient is a few numbers, each a sum over every row and layer that can cancel to a small part of its terms
    (rnn.weight_hh at C = 1 cancelled to 1.8e-6 in one H100 run); 2^-20 of such a value is less than any fp32 summation of the rows
    promises.  As test_gpu_rows_envelope.py does for narrow models, the parameter gradients of such a model share one scale, the model's
    largest parameter gradient: the same reductions over the same rows.  Where the LSTM stage is cuDNN's, its rounding reaches the fused side and the
    yardstick through different inputs and does not cancel: C = 31 on 4 225 nodes reached 4.98x e32 on one run and not on another, so
    those cases are allowed 8x."""
    n, fam = X.size(0), f"ggc_rows {c['aggr']}"
    gen = torch.Generator(device=DEV).manual_seed(seed)
    S = [0.5 * torch.randn(n, c["Ho"], device=DEV, generator=gen) for _ in range(2)]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]

    def oracle(dtype):
        p = {k: v.detach().to(dtype, copy=True).requires_grad_(True) for k, v in m.named_parameters()}
        x, h, cc = (t.to(dtype, copy=True).requires_grad_(True) for t in [X] + S)
        args = (p, c, x, ei, None if ew is None else ew.to(dtype), h if given else None, cc if given else None)
        o = dygrae_step(*args) if dtype == torch.float64 else _yardstick(m, *args)
        return list(o), [x, h, cc] + [p[k] for k in names]
    with _float64():
        o64, l64 = oracle(torch.float64)
    o32, l32 = oracle(torch.float32)
    wgts = [torch.randn(o.shape, device=DEV, generator=gen) for o in o64]
    state = S if given else [None, None]
    with torch.no_grad(), _counted() as cnt:
        inf = m(X, ei, ew, *state)
    assert _ran(cnt) == _dy_launches(c, False, False), (what, cnt)
    if not train:
        for i in range(3):
            _check_err(errs, fam, inf[i], o32[i], o64[i], what + (OUTS[i],))
        return
    g64 = _loss_grads(o64, [w.double() for w in wgts], l64)
    g32 = _loss_grads(o32, wgts, l32)
    xf = X.clone().requires_grad_(want_dx)
    sf = [s.clone().requires_grad_(True) for s in S] if given else [None, None]
    m.zero_grad(set_to_none=True)
    with _counted() as cnt:
        of = m(xf, ei, ew, *sf)
        gf = _loss_grads(list(of), wgts, [xf] + sf + params)
    assert _ran(cnt) == _dy_launches(c, True, want_dx), (what, cnt)
    if _rows_lstm(c):                            # (cuDNN's training and inference LSTM kernels may round differently)
        assert all(torch.equal(a.detach(), b) for a, b in zip(of, inf)), (what, "training forward differs from inference")
    for i in range(3):
        _check_err(errs, fam, of[i], o32[i], o64[i], what + (OUTS[i],))
    gscale = max(float(g.abs().max()) for g in g64[3:]) if c["C"] <= 2 else None
    for label, want, got, r32, r64 in zip(["dX", "dH", "dC"] + names, [want_dx, given, given] + [True] * len(names), gf, g32, g64):
        if not want:
            assert got is None, (what, label, "unwanted gradient")
            continue
        assert got is not None, (what, label)
        _check_err(errs, fam, got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (label,), 4 if _rows_lstm(c) else 8,
                   gscale if label in names else None)


def _contract(m, f):
    """Scales the convolution's weights by f.  A deep stack of N(0, 0.4) layers at C ~ 32 is a chaotic map that amplifies one rounding
    by ~1e4 over 33 layers (errors of 1e4 on gradients of 4e4 in one run), where float32 and float64 no longer compare; scaled, the layers
    contract."""
    with torch.no_grad():
        for q in m.conv_layer.parameters():
            q.mul_(f)
    return m


def _dy_graph(kind, n, seed=0):
    """(edge_index, the make_graph triple or None): make_graph's kinds; "holes": random with no in-edge into the last three rows and row
    n // 2; "E0": no edge."""
    if kind == "E0":
        return torch.zeros(2, 0, dtype=torch.int64, device=DEV), None
    g = make_graph("random" if kind == "holes" else kind, n, seed)
    src, dst, _ = g
    if kind == "holes":
        keep = (dst < n - 3) & (dst != n // 2)
        src, dst, g = src[keep], dst[keep], None
    return torch.from_numpy(np.stack([src, dst])).to(DEV), g


def _dy_weights(kind, E, seed):
    w = _weights(kind, E, seed)
    return None if w is None else w.to(DEV)


DY_CONFIGS = [(C, cin) for C in (1, 2, 15, 16, 17, 31, 32) for cin in sorted({1, C - 1, C}) if cin >= 1]   # C 16 | 17: row-split | cuDNN LSTM
LAYERS = (1, 2, 3, 8, 33)
WEIGHTS = (None, "pos", "signed")
# N: one warp's rows and 16-row tiles on either side of their edges, the weight gradient's 32-row tiles (a tile spans two layers whenever
# N % 32 != 0 and L_g >= 2), and 4 225 rows, where the grid stride starts; graphs: a ring (the gather's 4-unrolled body never runs),
# every in- and every out-degree residue mod 4, an in-hub and an out-hub of N - 1 edges, duplicates, a node without out-edges, rows
# without in-edges, E = 0.
DY_GEOMETRIES = ([("ring", n) for n in (1, 2, 15, 16, 17, 31, 32, 33)]
                 + [("mod4", 129), ("mod4_out", 129), ("hubs", 130), ("dups", 97), ("sink", 65), ("holes", 96), ("E0", 9), ("mod4", 4224),
                    ("hubs", 4225)])


@pytest.mark.parametrize("kind,n", DY_GEOMETRIES, ids=[f"{k}-N{n}" for k, n in DY_GEOMETRIES])
def test_geometries_against_float64(kind, n):
    """add and mean: every (C, cin) on every geometry, L_g, the edge weights, lstm_out_channels, H / C given and dX wanted cycling so that
    each meets each; two LSTM layers now and then (the cuDNN stage).  max: test_max_*."""
    gi = DY_GEOMETRIES.index((kind, n))
    ei, g = _dy_graph(kind, n, gi)
    errs = []
    for idx, (C, cin) in enumerate(DY_CONFIGS):
        s = idx + gi
        aggr = ("add", "mean")[idx % 2]
        wk = WEIGHTS[(idx // 2 + gi) % 3]
        c = dict(C=C, Lg=LAYERS[s % 5], aggr=aggr, Ho=(32, 64)[(idx // 3 + gi) % 2], Ll=2 if s % 7 == 3 else 1)
        m = _model(C, c["Lg"], aggr, c["Ho"], idx + n, c["Ll"]).to(DEV)
        if c["Lg"] >= 8:
            _contract(m, min(0.5, 1.5 / C ** 0.5))
        if idx == 0 and g is not None:
            check_family(kind, n, g, _Relation(m._plan(ei, None, n), 0), cheb=False)
        ew = _dy_weights(wk, ei.size(1), s)
        X = torch.randn(n, cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(s))
        given = bool(s >> 1 & 1) and c["Ll"] == 1            # a one-layer (N, Ho) state does not feed a two-layer LSTM (test_carried_state_errors)
        _dy_case(errs, m, c, X, ei, ew, given, s % 3 != 0, 31 * n + idx, (kind, n, C, cin, c["Lg"], aggr, wk, c["Ho"], c["Ll"]))
    assert not errs, errs[:6]


# (C, F, L_g) -> k: the max case of test_envelope_against_float64 draws X and the edge weights from seed + 1000 k, chosen so that its
# float64 forward has no near-tie (_max_gap); k = 0 elsewhere
MAX_RESEED = {(4, 1, 3): 2, (16, 1, 3): 2, (17, 1, 3): 1, (32, 1, 1): 1, (32, 1, 2): 1, (32, 32, 3): 1, (32, 1, 3): 1}


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("C", [1, 4, 5, 16, 17, 32])
@pytest.mark.parametrize("Fk", ["one", "full"])
@pytest.mark.parametrize("Lg", [1, 2, 3])
def test_envelope_against_float64(aggr, C, Fk, Lg):
    """Every aggregation x C x in_channels 1 or C x L_g on 37 nodes with duplicates, self loops and rows without in-edges, the weights,
    lstm_out_channels, the state and dX cycling; held to the criterion with its launches.  max takes seeds whose float64 forward keeps
    every top-two gap of a row at least 2^-16 of its layer's largest message (MAX_RESEED), asserted before the comparison."""
    F = 1 if Fk == "one" else C
    seed = 100 * C + 10 * Lg + F + AGGRS.index(aggr)
    Ho = (32, 64)[seed % 2]
    wk = (None, "pos", "signed")[seed % 3]
    with_state = (seed // 3) % 2 == 0
    n = 37
    ei = _graph_of("random", n, seed).to(DEV)
    xs = seed + 1000 * MAX_RESEED.get((C, F, Lg), 0) if aggr == "max" else seed
    ew = _dy_weights(wk, ei.size(1), xs)
    X = torch.randn(n, F, generator=torch.Generator().manual_seed(xs)).to(DEV)
    c = dict(C=C, Lg=Lg, aggr=aggr, Ho=Ho, Ll=1)
    m = _model(C, Lg, aggr, Ho, seed).to(DEV)
    if aggr == "max":
        assert _max_gap(m, X, ei, ew, C, Lg) >= 2.0 ** -16, "a near-tie: choose another X seed"
    errs = []
    _dy_case(errs, m, c, X, ei, ew, with_state, seed % 4 != 0, seed, (aggr, C, F, Lg, Ho, wk, with_state))
    assert not errs, errs[:6]


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("kind,n", [("empty", 9), ("one_node", 1), ("hub", 1200), ("random", 50000)])
def test_graph_geometries(aggr, kind, n):
    """0 edges, one node, rows without in-edges, a 400-edge hub and source, duplicate edges, self loops and 50 000 nodes, held to the
    criterion with the launches.  max runs at L_g = 1 on dyadic X, W_0 and edge weights (as _dyadic_case), where every message is exact
    in float32 and float64: duplicates are exact ties whose gradient split (torch's tie count) is compared like every other value, and no
    near-tie can swap an argmax between the two precisions.  On the hub, add and mean are held to the criterion with positive weights; with
    signed ones the hub row sums 400 cancelling messages, whose rounding in either path grows with the row while the yardstick's
    (index_add's atomics) changes from run to run, and reached 9x it once, so that case keeps the 1e-3 relative bound of _check_step."""
    ei = _graph_of(kind, n, 7).to(DEV)
    C, Ho, F = 16, 32, 14
    c = dict(C=C, Lg=1 if aggr == "max" else 2, aggr=aggr, Ho=Ho, Ll=1)
    if aggr == "max":
        rng = np.random.default_rng([n, 7])
        X = torch.from_numpy(rng.integers(-8, 9, (n, F)) / 8.0).float().to(DEV)
        ew = torch.from_numpy(rng.choice(DYADIC_W["signed"], ei.size(1))).float().to(DEV) if kind == "hub" else None
        m = _dyadic_model(C, Ho, n)
    else:
        if kind == "hub":           # signed weights on the 400-edge hub: held to the row-split tolerance of the goldens, see below
            gen = torch.Generator().manual_seed(n)
            Xs, Hs, Cs = torch.randn(n, F, generator=gen), torch.randn(n, Ho, generator=gen) * 0.5, torch.randn(n, Ho, generator=gen) * 0.5
            _check_step(_model(C, 2, aggr, Ho, n), c, Xs, ei.cpu(), _weights("signed", ei.size(1), 7), Hs, Cs, want_dx=True)
        ew = _dy_weights("pos" if kind == "hub" else None, ei.size(1), 7)
        X = torch.randn(n, F, generator=torch.Generator().manual_seed(n)).to(DEV)
        m = _model(C, 2, aggr, Ho, n).to(DEV)
    errs = []
    _dy_case(errs, m, c, X, ei, ew, True, True, n, (aggr, kind, n))
    assert not errs, errs[:6]


def test_carried_recurrence_vs_float64():
    """Five steps with H and C fed back and one backward through all of them (the row-split LSTM stage, mean aggregation, two layers)."""
    n, C, cin, steps = 129, 16, 13, 5
    c = dict(C=C, Lg=2, aggr="mean", Ho=32, Ll=1)
    ei, _ = _dy_graph("mod4_out", n)
    ew = _dy_weights("signed", ei.size(1), 3)
    m = _model(C, 2, "mean", 32, 11).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(2)
    X = torch.randn(steps, n, cin, device=DEV, generator=gen)
    S0 = [0.5 * torch.randn(n, 32, device=DEV, generator=gen) for _ in range(2)]
    wgts = [torch.randn(n, 32, device=DEV, generator=gen) for _ in range(2 * steps)]
    names = [k for k, _ in m.named_parameters()]

    def run_(dtype, step):
        x = X.to(dtype, copy=True).requires_grad_(True)
        s0 = [s.to(dtype, copy=True).requires_grad_(True) for s in S0]
        state, outs = s0, []
        for t in range(steps):
            o = step(x[t], state)
            state = list(o[1:])
            outs += [o[0], o[2]]
        return x, s0, outs
    g = {}
    for dtype in (torch.float64, torch.float32):
        p = {k: v.detach().to(dtype, copy=True).requires_grad_(True) for k, v in m.named_parameters()}
        wd = ew.to(dtype)
        with _float64() if dtype == torch.float64 else contextlib.nullcontext():
            x, s0, o = run_(dtype, lambda xt, st: dygrae_step(p, c, xt, ei, wd, *st))
        g[dtype] = [torch.stack(o)] + _loss_grads(o, [w.to(dtype) for w in wgts], [x] + s0 + [p[k] for k in names])
    m.zero_grad(set_to_none=True)
    with _counted() as cnt:
        xf, sf, of = run_(torch.float32, lambda xt, st: m(xt, ei, ew, *st))
        gf = [torch.stack(of)] + _loss_grads(of, wgts, [xf] + sf + [p for _, p in m.named_parameters()])
    assert _ran(cnt) == {k: steps * v for k, v in _dy_launches(c, True, True).items()}, cnt
    errs = []
    for label, got, r32, r64 in zip(["out", "dX", "dH0", "dC0"] + names, gf, g[torch.float32], g[torch.float64]):
        _check_err(errs, "ggc_rows mean", got, r32, r64, ("recurrence", label))
    assert not errs, errs[:6]


@pytest.mark.parametrize("aggr,Lg", [("add", 1024), ("mean", 1024), ("add", 1025), ("mean", 1025), ("max", 1025)])
def test_the_layer_limit(aggr, Lg):
    """stmp_ggc_rows_* take up to 1 024 layers.  At 1 024 the row-split kernels serve inference; at 1 025 the module runs op for op
    (no row-split launch, for inference and training alike) and matches float64, its LSTM stage the module's cuDNN LSTM.  Outputs only: at max, a thousand layers of random
    messages hold near-ties that float32 and float64 break differently, which moves gradients but not values."""
    n, C, cin = 33, 8, 5
    c = dict(C=C, Lg=Lg, aggr=aggr, Ho=32, Ll=1)
    ei, _ = _dy_graph("mod4", n)
    ew = _dy_weights("pos", ei.size(1), 1)
    m = _contract(_model(C, Lg, aggr, 32, Lg).to(DEV), 0.25)
    X = torch.randn(n, cin, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    errs = []
    if Lg <= 1024:
        _dy_case(errs, m, c, X, ei, ew, True, False, 5, (aggr, Lg), train=False)
        assert not errs, errs
        return
    gen = torch.Generator(device=DEV).manual_seed(5)
    H, Cs = (0.5 * torch.randn(n, 32, device=DEV, generator=gen) for _ in range(2))
    p = {k: v.detach() for k, v in m.named_parameters()}
    with _float64():
        o64 = dygrae_step({k: v.double() for k, v in p.items()}, c, X.double(), ei, ew.double(), H.double(), Cs.double())
    o32 = _yardstick(m, p, c, X, ei, ew, H, Cs, cudnn=True)
    for grad in (False, True):
        with torch.set_grad_enabled(grad), _counted() as cnt:
            o = m(X, ei, ew, H, Cs)
            if grad:
                o[0].sum().backward()
        assert _ran(cnt) == {}, (aggr, Lg, grad, cnt)
        for i in range(3):
            _check_err(errs, f"ggc_rows {aggr}", o[i], o32[i], o64[i], (aggr, Lg, grad, OUTS[i]))
    assert not errs, errs


# ---- max: compared where float32 and float64 agree on the argmax ----------------------------------------------------------------------
DYADIC_W = {None: None, "pos": (0.5, 1.0, 2.0), "signed": (0.0, 0.5, -0.5, 1.0, -1.0, 2.0, -2.0)}


def _dyadic_case(n, cin, wk, seed):
    """(edge_index, edge_weight, X) on which every message x W_0 and every w m is exact in float32 and float64 (X and W_0 of k / 8, |k| <= 8,
    at most 16 terms; weights from {0, ±1/2, ±1, ±2}), destination i by i % 14: no in-edge (0); in-degree 1..9 (1..9); one edge three
    times plus another (10: exact ties of a duplicated edge); three messages of exactly 0 (11: zero weights, or zero-X sources without
    signed weights); one edge from a zero-X source (12: a maximum of -0.0 at a negative weight, else +0.0); two or three distinct sources
    with the same X row and weight (13: exact ties between distinct sources)."""
    rng = np.random.default_rng([seed, n, cin])
    X = rng.integers(-8, 9, (n, cin)) / 8.0
    nodes = np.arange(n)
    zero = nodes[nodes % 19 == 1]
    twin = nodes[(nodes % 17 == 5) & (nodes % 19 != 1)]
    X[zero] = 0.0
    X[twin] = X[twin[0]] if twin.size else 0.0
    ws = DYADIC_W[wk] or (1.0,)
    src, dst, w = [], [], []
    for i in range(n):
        p = i % 14
        if p == 0:
            continue
        if 1 <= p <= 9:
            s, e = rng.integers(0, n, p), rng.choice(ws, p)
        elif p == 10:
            j, k, a = rng.integers(0, n, 2).tolist() + [rng.choice(ws)]
            s, e = np.array([j, j, k, j]), np.array([a, a, rng.choice(ws), a])
        elif p == 11:
            s = rng.integers(0, n, 3) if wk == "signed" else rng.choice(zero, 3)
            e = np.zeros(3) if wk == "signed" else rng.choice(ws, 3)
        elif p == 12:
            s, e = rng.choice(zero, 1), np.array([-0.5 if wk == "signed" else ws[0]])
        else:
            k = 2 + i % 2
            s, e = rng.choice(twin, k, replace=twin.size < k), np.full(k, rng.choice(ws))
        src.append(s)
        dst.append(np.full(s.size, i))
        w.append(e)
    src, dst, w = (np.concatenate(a) if a else np.zeros(0) for a in (src, dst, w))
    ei = torch.from_numpy(np.stack([src, dst]).astype(np.int64)).to(DEV)
    ew = None if wk is None else torch.from_numpy(w).float().to(DEV)
    return ei, ew, torch.from_numpy(X).float().to(DEV)


def _dyadic_model(C, Ho, seed):
    m = _model(C, 1, "max", Ho, seed)
    with torch.no_grad():
        g = torch.Generator().manual_seed(seed)
        m.conv_layer.weight.copy_(torch.randint(-8, 9, (1, C, C), generator=g) / 8.0)
    return m.to(DEV)


@pytest.mark.parametrize("wk", WEIGHTS)
def test_max_exact_ties_and_zeros_vs_float64(wk):
    """L_g = 1 on dyadic inputs (_dyadic_case): every maximum, every tie and every tie count is the same in float32 and float64, so the
    split of a row's gradient over its tied messages -- torch's scatter_reduce("amax", include_self=False): the count of messages equal to
    the maximum, one more when it is exactly 0 -- is held to the criterion with the rest."""
    n = 14 * 5
    errs = []
    for idx, (C, cin) in enumerate([(1, 1), (4, 3), (4, 4), (15, 1), (15, 14), (16, 16), (16, 15)]):
        ei, ew, X = _dyadic_case(n, cin, wk, idx)
        m = _dyadic_model(C, (32, 64)[idx % 2], idx)
        c = dict(C=C, Lg=1, aggr="max", Ho=(32, 64)[idx % 2], Ll=1)
        _dy_case(errs, m, c, X, ei, ew, bool(idx % 3), idx % 2 == 0, idx, ("dyadic", wk, C, cin))
    assert not errs, errs[:6]


def test_max_exact_ties_on_a_50000_node_graph_vs_float64():
    n = 50000
    errs = []
    for idx, (C, cin, wk) in enumerate([(16, 16, "signed"), (8, 5, None), (15, 15, "pos")]):
        ei, ew, X = _dyadic_case(n, cin, wk, 100 + idx)
        c = dict(C=C, Lg=1, aggr="max", Ho=32, Ll=1)
        _dy_case(errs, _dyadic_model(C, 32, idx), c, X, ei, ew, True, True, idx, ("dyadic 50000", wk, C, cin))
    assert not errs, errs[:6]


def _max_gap(m, X, ei, ew, C, L):
    """The smallest gap, over rows, channels and layers, between the largest and the second-largest distinct message w_e m_j of a row
    (exact duplicates excluded), relative to that layer's largest message; the float64 forward of GatedGraphConv."""
    p = {k: v.detach().double() for k, v in m.conv_layer.named_parameters()}
    x = torch.cat([X.double(), X.new_zeros(X.size(0), C - X.size(1), dtype=torch.float64)], 1)
    src, dst = ei[0], ei[1]
    w = torch.ones(ei.size(1), dtype=torch.float64, device=X.device) if ew is None else ew.double()
    idx = dst.view(-1, 1).expand(-1, C)
    worst = float("inf")
    for W in p["weight"][:L]:
        msg = w.view(-1, 1) * (x @ W)[src]
        if msg.numel():
            top = msg.new_zeros(x.shape).scatter_reduce(0, idx, msg, "amax", include_self=False)
            below = torch.where(msg < top[dst], msg, torch.full_like(msg, -float("inf")))
            second = torch.full_like(x, -float("inf")).scatter_reduce(0, idx, below, "amax", include_self=True)
            gap = (top - second)[torch.isfinite(second)]
            if gap.numel():
                worst = min(worst, float(gap.min()) / float(msg.abs().max()))
        x = gru_cell(aggregate(x @ W, ei, w, "max"), x, p["rnn.weight_ih"], p["rnn.weight_hh"], p["rnn.bias_ih"], p["rnn.bias_hh"])
    return worst


# (kind, N, C, cin, L_g, lstm_out_channels, weights, seed): random inputs whose float64 forward keeps every top-two gap of a max at
# least 2^-16 of its layer's largest message, so no argmax can swap between float32 and float64 (the seeds were chosen for that).
MAX_CASES = [("mod4", 33, 4, 3, 2, 32, "signed", 0), ("random", 17, 16, 16, 3, 64, None, 0), ("dups", 40, 17, 1, 8, 32, "pos", 1),
             ("hubs", 33, 2, 1, 33, 32, "signed", 2), ("mod4_out", 129, 8, 8, 2, 64, "pos", 0), ("mod4", 31, 32, 31, 2, 32, None, 1),
             ("random", 4225, 1, 1, 2, 32, "signed", 94), ("mod4", 4224, 1, 1, 2, 64, None, 2)]


def _max_inputs(case):
    kind, n, C, cin, Lg, Ho, wk, seed = case
    ei, _ = _dy_graph(kind, n, seed)
    m = _model(C, Lg, "max", Ho, 1000 * seed + n + C).to(DEV)
    X = torch.randn(n, cin, generator=torch.Generator().manual_seed(seed)).to(DEV)
    return m, X, ei, _dy_weights(wk, ei.size(1), seed)


@pytest.mark.parametrize("case", MAX_CASES, ids=[f"{k}-N{n}-C{C}-L{L}" for k, n, C, _, L, *_ in MAX_CASES])
def test_max_screened_vs_float64(case):
    """max at L_g >= 2 on random inputs screened for near-ties: gather_max's 4-unrolled body and tail over every degree residue, hubs,
    duplicates (exact ties), a weight-gradient tile spanning two layers (N % 32 != 0)."""
    kind, n, C, cin, Lg, Ho, wk, seed = case
    m, X, ei, ew = _max_inputs(case)
    assert _max_gap(m, X, ei, ew, C, Lg) >= 2.0 ** -16, "a near-tie: choose another seed"
    c = dict(C=C, Lg=Lg, aggr="max", Ho=Ho, Ll=1)
    errs = []
    for given, want_dx in ((False, True), (True, False)):
        _dy_case(errs, m, c, X, ei, ew, given, want_dx, n + given, case + (given, want_dx))
    assert not errs, errs[:6]


@pytest.mark.parametrize("parts", [1, 7, 8, 9, "full"])
@pytest.mark.parametrize("C,L", [(5, 3), (32, 2)])
def test_ggc_wgrad_reduce_is_the_fixed_order_sum(C, L, parts):
    """stmp_ggc_rows_wgrad: k_ggc_rows_wgrad (one partial of kWgPart = 3 168 floats per (job, CTA) over 32-row tiles of the L N rows), then
    k_ggc_rows_wgrad_reduce over its job layout: dW_ih | db_ih (job 0), dW_hh | db_hh (job 1), dW_l (job 2 + l); every element
    recomputed in float32 in the reduce's association (test_gpu_wgrad_reduce.py)."""
    torch.manual_seed(C + L)
    cap = 2 * _sms()
    n = _rows(parts, 32, cap) // L
    k = _parts(L * n, 32, cap)
    assert k == (cap if parts == "full" else parts)
    ring = torch.arange(n, device=DEV)
    plan = GatedPlan(torch.stack([ring, (ring + 1) % n]), None, n, "add")
    stash, dG, dM = _randn(L, 8, n, C), _randn(L, n, 4 * C), _randn(L, n, C)
    ws = _workspace(_lib.lib().stmp_ggc_rows_wgrad_workspace_bytes(L, C))
    out = [torch.full(s, NAN, device=DEV) for s in ((L, C, C), (3 * C, C), (3 * C, C), (3 * C,), (3 * C,))]
    with _counted() as cnt:
        _check(_lib.lib().stmp_ggc_rows_wgrad(plan.handle, L, C, _lib.ptr(stash), _lib.ptr(dG), _lib.ptr(dM), _lib.ptr(ws),
                                              *(_lib.ptr(t) for t in out), _lib.stream_ptr()))
    assert _ran(cnt) == {"k_ggc_rows_wgrad": 1, "k_ggc_rows_wgrad_reduce": 1}, cnt
    part = 3 * 32 * 32 + 3 * 32
    P = ws[:(2 + L) * k * part].view(2 + L, k, part).cpu()
    dW, dwih, dwhh, dbih, dbhh = out
    _equal(dwih, _sum(P[0], _ar(3 * C * C).view(3 * C, C)))
    _equal(dbih, _sum(P[0], 3 * 32 * 32 + _ar(3 * C)))
    _equal(dwhh, _sum(P[1], _ar(3 * C * C).view(3 * C, C)))
    _equal(dbhh, _sum(P[1], 3 * 32 * 32 + _ar(3 * C)))
    for l in range(L):
        _equal(dW[l], _sum(P[2 + l], _ar(C * C).view(C, C)))


@pytest.mark.parametrize("aggr", AGGRS)
def test_exact_ties_split_the_gradient(aggr):
    """Every edge appears three times: each max is an exact three-way tie in float32 and float64 alike."""
    ei = _graph_of("random", 50, 3)
    ei = torch.cat([ei, ei, ei], 1)
    g = torch.Generator().manual_seed(4)
    X = torch.randn(50, 8, generator=g)
    c = dict(C=8, Lg=2, aggr=aggr, Ho=32, Ll=1)
    _check_step(_model(8, 2, aggr, 32, 5), c, X, ei, None, None, None, want_dx=True)


def _launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, _lib.launch_count() - n0


@pytest.mark.parametrize("aggr", AGGRS)
@pytest.mark.parametrize("Lg", [1, 3])
def test_training_equals_inference_repeats_and_counts(aggr, Lg):
    """Inference and the training forward: L_g GatedGraphConv launches (one more for max) + one LSTM launch.  Backward: the LSTM cell's
    one + two weight-gradient launches, then L_g GatedGraphConv launches, one more for dX (add, mean) or always (max), and two for its
    weight gradients."""
    m = _model(16, Lg, aggr, 32, 3).to(DEV)
    ei = _graph_of("hub", 700, 3).to(DEV)
    ew = _weights("pos", ei.size(1), 3).to(DEV)
    g = torch.Generator().manual_seed(2)
    X, H, C = torch.randn(700, 14, generator=g).to(DEV), torch.randn(700, 32, generator=g).to(DEV), torch.randn(700, 32, generator=g).to(DEV)
    mx = aggr == "max"
    with torch.no_grad():
        want = m(X, ei, ew, H, C)
        got, n = _launches(lambda: m(X, ei, ew, H, C))
    assert n == Lg + mx + 1
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    out, n = _launches(lambda: m(X, ei, ew, H, C))
    assert n == Lg + mx + 1
    assert all(torch.equal(a, b) for a, b in zip(out, want))
    for want_dx in (False, True):
        Xg = X.clone().requires_grad_(want_dx)
        grads = []
        for scale in (1.0, 1.0, 8.0):
            m.zero_grad()
            o = m(Xg, ei, ew, H, C)
            loss = (o[0].square().mean() + o[2].mean()) * scale
            _, n = _launches(lambda: loss.backward())
            assert n == 3 + Lg + (1 if (mx or want_dx) else 0) + 2
            grads.append([p.grad.clone() for p in m.parameters()] + ([Xg.grad.clone()] if want_dx else []))
            if want_dx:
                Xg.grad = None
        assert all(torch.equal(a, b) for a, b in zip(grads[0], grads[1]))
        assert all(torch.equal(a * 8, b) for a, b in zip(grads[0], grads[2]))


@pytest.mark.parametrize("C,Ll,dtype,conv,lstm", [(20, 1, torch.float32, True, False), (8, 2, torch.float32, True, False),
                                                  (8, 1, torch.float64, False, False), (8, 1, torch.float32, True, True)])
def test_routes(C, Ll, dtype, conv, lstm):
    """C in 17..32 or two LSTM layers: the row-split convolution feeds the module's cuDNN LSTM; float64: op for op."""
    torch.manual_seed(0)
    m = DyGrEncoder(C, 2, "mean", 32, Ll).to(DEV).to(dtype)
    ei = _graph_of("random", 200, 1).to(DEV)
    X = torch.randn(200, 6, device=DEV, dtype=dtype)
    before = dict(_lib.path_counters())
    with torch.no_grad():
        h, H, Cc = m(X, ei)
    after = _lib.path_counters()
    assert (after.get("k_ggc_rows_fwd", 0) > before.get("k_ggc_rows_fwd", 0)) is conv
    assert (after.get("k_lstm_rows_fwd", 0) > before.get("k_lstm_rows_fwd", 0)) is lstm
    p64 = _params64(m)
    want = dygrae_step(p64, dict(C=C, Lg=2, aggr="mean", Ho=32, Ll=Ll), X.double().cpu(), ei.cpu(), None)
    for a, b, what in zip((h, H, Cc), want, ("H_tilde", "H", "C")):
        _close(a, b, what, 1e-4)
    assert h.data_ptr() != H.data_ptr()


def test_carried_state_errors():
    m = DyGrEncoder(4, 1, "mean", 32, 1).to(DEV)
    x, ei = torch.randn(1, 3, device=DEV), torch.zeros(2, 0, dtype=torch.int64, device=DEV)
    _, H, C = m(x, ei)
    assert H.shape == (32,)
    with pytest.raises(IndexError):
        m(x, ei, None, H, C)
    m = DyGrEncoder(4, 1, "mean", 32, 2).to(DEV)
    x, ei = torch.randn(5, 3, device=DEV), torch.tensor([[0, 1], [1, 2]], device=DEV)
    _, H, C = m(x, ei)
    with pytest.raises(RuntimeError):
        m(x, ei, None, H, C)
    with pytest.raises(RuntimeError):                       # batched X is not supported by the reference either
        m(torch.randn(2, 5, 3, device=DEV), ei)


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
    gp = GatedPlan(ei.to(DEV), ew.to(DEV), 20, "max")
    assert L.stmp_ggc_rows_supported(gp.handle, 3, 4, 32) == 1
    assert L.stmp_ggc_rows_supported(gp.handle, 1, 33, 33) == 0
    assert L.stmp_ggc_rows_supported(gp.handle, 1, 5, 4) == 0
    assert L.stmp_ggc_rows_supported(gp.handle, 0, 4, 4) == 0
    assert L.stmp_ggc_rows_supported(cheb.handle, 1, 4, 4) == 0
    assert L.stmp_lstm_rows_supported(gp.handle, _lib.LSTM_GCONV, 0, 16, 32) == 1
    assert L.stmp_lstm_rows_supported(gp.handle, _lib.LSTM_GCONV, 0, 16, 64) == 1
    buf = torch.zeros(1 << 20, device=DEV)
    p = _lib.ptr(buf)
    fwd = lambda plan, L_, cin, C: L.stmp_ggc_rows_fwd(plan, L_, cin, C, p, p, p, p, p, p, p, p, None, None)
    assert fwd(cheb.handle, 1, 4, 4) == _lib.STMP_EINVAL
    assert fwd(None, 1, 4, 4) == _lib.STMP_EINVAL
    assert fwd(gp.handle, 1, 5, 4) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_ggc_rows_fwd(gp.handle, 1, 4, 4, p, p, p, p, p, p, None, p, None, None) == _lib.STMP_EINVAL
    assert L.stmp_ggc_rows_bwd(gp.handle, 1, 4, 4, p, None, p, p, p, p, p, p, None, None) == _lib.STMP_EINVAL
    assert L.stmp_ggc_rows_wgrad(gp.handle, 1, 4, p, p, p, p, p, p, p, p, None, None) == _lib.STMP_EINVAL
    assert L.stmp_ggc_rows_wgrad_workspace_bytes(2, 32) > 0 and L.stmp_ggc_rows_wgrad_workspace_bytes(2, 33) == 0
    assert L.stmp_ggc_rows_scratch_bytes(gp.handle, 8) == 4 * 20 * 8 * 4
    torch.cuda.synchronize()
