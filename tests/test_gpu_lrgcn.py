"""LRGCN on the H100: the relational plans bit-exact against a CPU restatement, every golden case on the row-split cell and op for op against
the float64 oracle (held to the reference's fingerprints by tests/test_lrgcn_cpu.py), the envelope against float64, bit-equal training and
inference forwards, launch counts, the two-operator weight-gradient reduce bit for bit, routing outside the envelope and the ABI's errors.

Envelope criterion (test_gpu_rows_envelope.py's): lrgcn_cell in float64 on the GPU with autograd is the reference, lrgcn_cell in float32
(no TF32) the yardstick; every tensor -- H', C', each wanted dX / dH / dC and each parameter's gradient on its own -- stays within 4x the
yardstick's error plus 2^-20 of its scale, and a parameter gradient that is exactly 0 in float64 (a relation without edges) is exactly 0.
The basis coefficients' gradient takes the scale of its terms (_lrgcn_case).  Every case asserts the row-split launches of inference and
training (k_lstm_rows_* with the two-operator k_lstm_rows_wgrad2 at R = 2, k_dcrnn_wgrad at R = 1, k_lstm_wide_rows_* at 64 channels).
Shapes: every cin 1..16 at R = 2 (nb = 3 (cin + 32): cin 10 | 11 is the backward's fifth 32-column group, cin 16 fills dS's scratch row),
R = 1 and 64 channels, num_bases None / 1 / 2 / 3; N 1, 2, 15, 16, 17, 33, 129, 207, 4 224, 4 225 (the forward's grid stride) and 50 000;
per relation a ring, every in- and out-degree residue mod 4, in- and out-hubs of N - 1 edges, duplicates, a node with in-edges of the
other relation only, relation 1 empty, both empty, E = 0, and edges whose type selects no relation; H and C None or given, dX, dH and dC
each wanted or not; a 5-step carried sequence.

Largest ratios of one run on an H100 80GB HBM3 at a 700 W power limit, as printed by `_report` (`e / e32` over comparisons above the
2^-20 floor; `used`: the largest fraction of the allowance consumed):
    lstm_rows R=1        e / e32 1.39   used 0.41
    lstm_rows R=2        e / e32 3.16   used 0.54
    lstm_wide_rows R=1   e / e32 5.17   used 0.67
This file and test_gpu_dygrae.py took 121 s together there.
"""
import contextlib
import ctypes
import itertools
import os

import numpy as np
import pytest
import torch

from lrgcn_seq import edge_types, load, lrgcn_cell, model_for, oracle_run, run, states_for
from gconvgru_seq import chickenpox_train_split
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import LRGCN
from pytorch_geometric_temporal_b200.nn.recurrent.lrgcn import RGCNParams
from pytorch_geometric_temporal_b200.plan import GraphPlan, RgcnPlan
from test_gpu_rows_envelope import WORST, _check_err, _counted, _float64, _loss_grads, _or_zeros, check_family, make_graph
from test_gpu_wgrad_reduce import _ar, _check, _equal, _operands, _parts, _randn, _rows, _sms, _sum, _workspace, PARTS, NAN
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


# ---- the envelope against float64 (the criterion of test_gpu_rows_envelope.py) -------------------------------------------------------
@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for fam in FAMILIES:
        if fam in WORST:
            ratio, used, what = WORST[fam]
            print(f"\nLRGCN envelope: {fam}: largest e / e32 = {ratio:.2f}, largest used fraction of the allowance = {used:.2f} at {what}")


@pytest.fixture(autouse=True)
def _fp32():
    """The fp32 yardstick (lrgcn_cell in float32 on the GPU) in full fp32: no TF32 in cuBLAS or cuDNN."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _family(R, co):
    return "lstm_wide_rows R=1" if co == 64 else f"lstm_rows R={R}"


FAMILIES = ("lstm_rows R=1", "lstm_rows R=2", "lstm_wide_rows R=1")
NO_RELATION = (-1, 2, 5)                       # edge types that select no relation (and type 1 selects none at R = 1)


def _launches(R, co, gather, train=True):
    """The row-split launches of one LRGCN step; `gather`: dX or dH wanted (k_lstm_rows_bwd_b gathers both operators' Op^T Q)."""
    if co == 64:
        want = {"k_lstm_wide_rows_fwd": 1}
        if train:
            want.update({"k_lstm_wide_rows_bwd_a": 1, "k_lstm_wide_rows_bwd_b": int(gather), "k_lstm_wide_rows_wgrad": 1,
                         "k_lstm_wide_rows_wgrad_reduce": 1})
    else:
        want = {"k_lstm_rows_fwd": 1}
        if train:
            want.update({"k_lstm_rows_bwd_a": 1, "k_lstm_rows_bwd_b": int(gather)})
            want.update({"k_lstm_rows_wgrad2": 1, "k_lstm_rows_wgrad2_reduce": 1} if R == 2 else
                        {"k_dcrnn_wgrad": 1, "k_lstm_rows_wgrad_reduce": 1})
    return {k: v for k, v in want.items() if v}


ROW_SPLIT = ("k_lstm_rows_fwd", "k_lstm_rows_bwd_a", "k_lstm_rows_bwd_b", "k_lstm_rows_wgrad2", "k_lstm_rows_wgrad2_reduce", "k_dcrnn_wgrad",
             "k_lstm_rows_wgrad_reduce", "k_lstm_wide_rows_fwd", "k_lstm_wide_rows_bwd_a", "k_lstm_wide_rows_bwd_b", "k_lstm_wide_rows_wgrad",
             "k_lstm_wide_rows_wgrad_reduce", "k_spmm")


def _ran(c):
    return {k: v for k, v in c.items() if k in ROW_SPLIT}


class _Relation:
    """Relation r of an RgcnPlan seen as check_family's DConv plan: operator 0 its CSR by destination, operator 1 the transposed one."""

    def __init__(self, plan, r):
        self.plan, self.r = plan, r

    def export(self, op, transposed=False):
        return self.plan.export(self.r, transposed != bool(op))


def _rel_graph(kinds, n, seed=0):
    """(edge_index, edge_type, per-relation graphs): relation r holds make_graph(kinds[r], n) (None: no edge), then edges of types that
    select no relation; the edges are shuffled so that relations interleave in every CSR row.  Node n // 3 keeps only relation 1's
    in-edges when both relations have edges (unless relation 0 is the hubs kind).  kinds = "E0": no edge at all."""
    if kinds == "E0":
        return torch.zeros(2, 0, dtype=torch.int64, device=DEV), torch.zeros(0, dtype=torch.int64, device=DEV), [None, None]
    rng = np.random.default_rng([seed, n])
    srcs, dsts, types, per = [], [], [], []
    for r, kind in enumerate(kinds):
        if kind is None:
            per.append(None)
            continue
        src, dst, _ = make_graph(kind, n, seed + r)
        if r == 0 and kind != "hubs" and kinds[1] is not None and n >= 3:      # (the out-hub keeps its N - 1 edges)
            keep = dst != n // 3
            src, dst = src[keep], dst[keep]
        per.append((src, dst, None))
        srcs.append(src)
        dsts.append(dst)
        types.append(np.full(src.size, r))
    src, dst, _ = make_graph("random", n, seed + 7)
    srcs.append(src)
    dsts.append(dst)
    types.append(rng.choice(NO_RELATION, src.size))
    src, dst, et = np.concatenate(srcs), np.concatenate(dsts), np.concatenate(types)
    order = rng.permutation(src.size)
    ei = torch.from_numpy(np.stack([src[order], dst[order]])).to(DEV)
    return ei, torch.from_numpy(et[order].astype(np.int64)).to(DEV), per


def _check_relations(m, kinds, n, ei, et, per):
    plan = m._relation_plans(ei, et, n)[0]
    for r in range(m.num_relations):
        if per[r] is None:
            assert all(int(t.numel()) == 0 for t in plan.export(r, False)[1:]), ("relation", r, "not empty")
        else:
            check_family(kinds[r], n, per[r], _Relation(plan, r), cheb=False)


def _lrgcn_model(cin, co, R, B, seed):
    torch.manual_seed(seed)
    m = LRGCN(cin, co, R, B).to(DEV)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("bias"):
                p.copy_(torch.randn_like(p) * 0.1)
    return m


def _lrgcn_case(errs, m, ei, et, n, given, wants, seed, what):
    """One LRGCN step on the row-split cell against float64: H', C' and every wanted gradient.  `given`: (H, C) passed (else None);
    `wants`: (dX, dH, dC) wanted.  Unwanted gradients must come back as None; a parameter gradient that is exactly 0 in float64 (a
    relation without edges, the H blocks of H = None) must be exactly 0.

    The basis coefficients' gradient dcomp[r, b] = <dW_r, V_b> is a dot product over in x out terms that cancel, down to 1e-4 of their
    sum of magnitudes; its error scale is that sum, max_{r,b} sum |dW_r| |V_b| (_comp_scales), not the cancelled value.  Against the
    cancelled value the yardstick's own error varies from run to run (index_add's atomics) down to 1e-13, and comp reached 55x it."""
    cin, co, R = m.in_channels, m.out_channels, m.num_relations
    fam = _family(R, co)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(n, cin, device=DEV, generator=gen)
    S = [0.5 * torch.randn(n, co, device=DEV, generator=gen) for _ in range(2)]
    wgts = [torch.randn(n, co, device=DEV, generator=gen) for _ in range(2)]
    wants = [wants[0], wants[1] and given[0], wants[2] and given[1]]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]

    def oracle(dtype):
        p = {k: v.detach().to(dtype, copy=True).requires_grad_(True) for k, v in m.named_parameters()}
        x, h, c = (t.to(dtype, copy=True).requires_grad_(True) for t in [X] + S)
        z = torch.zeros(n, co, dtype=dtype, device=DEV)
        o = lrgcn_cell(p, x, ei, et, h if given[0] else z, c if given[1] else z, R)
        return _loss_grads(list(o), [w.to(dtype) for w in wgts], [x, h, c] + [p[k] for k in names]), o
    with _float64():
        g64, o64 = oracle(torch.float64)
        comp_scale = _comp_scales(m, X, S, ei, et, given, wgts)
    g32, o32 = oracle(torch.float32)
    state = [S[i] if given[i] else None for i in range(2)]
    with torch.no_grad(), _counted() as c:
        inf = m(X, ei, et, *state)
    assert _ran(c) == _launches(R, co, False, train=False), (what, c)
    xf = X.clone().requires_grad_(wants[0])
    sf = [S[i].clone().requires_grad_(wants[1 + i]) if given[i] else None for i in range(2)]
    m.zero_grad(set_to_none=True)
    with _counted() as c:
        of = m(xf, ei, et, *sf)
        gf = _loss_grads(list(of), wgts, [xf] + sf + params)
    assert _ran(c) == _launches(R, co, wants[0] or wants[1]), (what, c)
    assert torch.equal(of[0].detach(), inf[0]) and torch.equal(of[1].detach(), inf[1]), (what, "training forward differs from inference")
    for i in range(2):
        _check_err(errs, fam, of[i], o32[i], o64[i], what + (("H'", "C'")[i],))
    for label, want, got, r32, r64 in zip(["dX", "dH", "dC"] + names, wants + [True] * len(names), gf, g32, g64):
        if not want:
            assert got is None, (what, label, "unwanted gradient")
            continue
        assert got is not None, (what, label)
        r64 = _or_zeros(r64, got.double())
        _check_err(errs, fam, got, _or_zeros(r32, got), r64, what + (label,), scale=comp_scale.get(label))
        if label in names:
            assert not bool(got[r64 == 0].any()), (what, label, "a structural zero of the gradient is not 0")


def _comp_scales(m, X, S, ei, et, given, wgts):
    """{"conv_*.comp": max over (r, b) of sum |dW_r| |V_b|} in float64, dW_r the gradient of relation r's weight W_r = sum_b comp[r, b] V_b
    (the relation weights taken as leaves); empty without bases."""
    if m.num_bases is None:
        return {}
    n, co, R = X.size(0), m.out_channels, m.num_relations
    p, V = {}, {}
    for k, conv in m.named_children():
        if not isinstance(conv, RGCNParams):
            continue
        p[f"{k}.weight"] = conv.relation_weights().detach().double().requires_grad_(True)
        p[f"{k}.root"], p[f"{k}.bias"] = conv.root.detach().double(), conv.bias.detach().double()
        V[k] = conv.weight.detach().double()
    z = torch.zeros(n, co, dtype=torch.float64, device=DEV)
    h, c = (S[i].double() if given[i] else z for i in range(2))
    o = lrgcn_cell(p, X.double(), ei, et, h, c, R)
    g = _loss_grads(list(o), [w.double() for w in wgts], [p[f"{k}.weight"] for k in V])
    return {f"{k}.comp": float(torch.einsum("rio,bio->rb", dW.abs(), V[k].abs()).max()) for k, dW in zip(V, g)}


# (cin, out, R, num_bases): every cin at R = 2 and R = 1 at 32 channels and at R = 1 at 64, the bases cycling.  R = 2: nb = 3 (cin + 32),
# so cin = 10 (nb 126) is the last basis without a fifth 32-column group in k_lstm_rows_bwd_a and cin = 11 (nb 129) the first with one;
# at cin = 16 dS's two operator blocks fill the 96-float scratch row.
CONFIGS = [(cin, co, R, (None, 1, 2, 3)[(cin + k) % 4]) for cin in range(1, 17) for k, (co, R) in enumerate(((32, 2), (32, 1), (64, 1)))]
# (relation kinds, N): a ring in relation 0 (one entry per row: the 4-unrolled gather body never runs), every in- and every out-degree
# residue mod 4 per relation, an in-hub and an out-hub of N - 1 edges, duplicates, relation 1 empty, both relations empty, E = 0; tiles
# of 16 rows, and 4 225 rows, where the forward's grid stride (2 x 132 CTAs of 16 rows) starts.
GEOMETRIES = ([(("ring", "random"), n) for n in (1, 2, 15, 16, 17, 33)]
              + [(("ring", None), 33), (("mod4", "mod4_out"), 207), (("mod4_out", "mod4"), 129), (("hubs", "dups"), 208),
                 (("dups", "hubs"), 129), ((None, None), 40), ("E0", 9), (("mod4", "dups"), 4224), (("mod4_out", "hubs"), 4225)])


@pytest.mark.parametrize("kinds,n", GEOMETRIES, ids=[f"{k if k == 'E0' else '-'.join(map(str, k))}-N{n}" for k, n in GEOMETRIES])
def test_geometries_against_float64(kinds, n):
    """Every (cin, out, R, num_bases) on every geometry; which of H and C are given and which of dX, dH, dC are wanted cycle."""
    assert 4225 > 2 * 132 * 16
    gi = GEOMETRIES.index((kinds, n))
    ei, et, per = _rel_graph(kinds, n, seed=gi)
    errs, checked = [], set()
    for idx, (cin, co, R, B) in enumerate(CONFIGS):
        s = idx + 3 * gi
        given = (bool(s & 1), bool(s >> 1 & 1))
        wants = (bool(s >> 2 & 1) or idx % 3 == 0, bool(s >> 3 & 1) or idx % 5 == 0, True)
        m = _lrgcn_model(cin, co, R, B, seed=idx + n)
        if R not in checked:
            _check_relations(m, kinds, n, ei, et, per)
            checked.add(R)
        _lrgcn_case(errs, m, ei, et, n, given, wants, 31 * n + idx, (kinds, n, cin, co, R, B, given, wants))
    assert not errs, errs[:6]


@pytest.mark.parametrize("R,B,co", [(1, None, 32), (1, 1, 32), (2, None, 32), (2, 1, 32), (2, 2, 32), (1, None, 64), (1, 2, 64)])
@pytest.mark.parametrize("cin", [1, 5, 16])
@pytest.mark.parametrize("n,with_state", [(1, True), (37, False), (1068, True), (50000, True)])
def test_envelope_against_float64(R, B, co, cin, n, with_state):
    """Relations x bases x width x cin on 1 to 50 000 nodes with a hub, rows without in-edges, duplicates, self loops and edges of a type
    that selects no relation; H and C given or None, every gradient wanted; held to the criterion with its launches (_lrgcn_case)."""
    m, ei, et, _, _, _ = _envelope_case(n, cin, co, R, B, with_state, n + cin + 7 * R)
    errs = []
    _lrgcn_case(errs, m.to(DEV), ei.to(DEV), et.to(DEV), n, (with_state, with_state), (True, True, True), n + cin + 7 * R,
                (n, cin, co, R, B, with_state))
    assert not errs, errs[:6]


@pytest.mark.parametrize("R,co", [(2, 32), (1, 32), (1, 64)])
def test_state_and_gradient_flags_vs_float64(R, co):
    """H and C each None or given, dX, dH and dC each wanted or not."""
    n = 33
    ei, et, _ = _rel_graph(("mod4", "mod4_out"), n, seed=3)
    m = _lrgcn_model(11, co, R, 2, seed=R)
    errs, seen = [], set()
    for given in itertools.product((False, True), repeat=2):
        for wants in itertools.product((False, True), repeat=3):
            eff = (given, (wants[0], wants[1] and given[0], wants[2] and given[1]))
            if eff in seen:
                continue
            seen.add(eff)
            _lrgcn_case(errs, m, ei, et, n, given, wants, len(seen), (R, co, given, wants))
    assert not errs, errs[:6]


def test_a_50000_node_graph_vs_float64():
    n = 50000
    ei, et, _ = _rel_graph(("mod4_out", "hubs"), n, seed=5)
    errs = []
    for cin, co, R, B in ((16, 32, 2, None), (11, 32, 2, 3), (10, 32, 2, 1), (5, 32, 1, None), (14, 64, 1, 2)):
        _lrgcn_case(errs, _lrgcn_model(cin, co, R, B, seed=cin), ei, et, n, (True, True), (True, True, True), cin, ("50000", cin, co, R, B))
    assert not errs, errs[:6]


@pytest.mark.parametrize("R,co", [(2, 32), (1, 64)])
def test_carried_recurrence_vs_float64(R, co):
    """Five steps with H and C fed back and one backward through all of them."""
    n, cin, steps = 129, 11, 5
    ei, et, _ = _rel_graph(("mod4", "mod4_out"), n, seed=9)
    m = _lrgcn_model(cin, co, R, 2, seed=11)
    gen = torch.Generator(device=DEV).manual_seed(2)
    X = torch.randn(steps, n, cin, device=DEV, generator=gen)
    S0 = [0.5 * torch.randn(n, co, device=DEV, generator=gen) for _ in range(2)]
    wgts = [torch.randn(n, co, device=DEV, generator=gen) for _ in range(2 * steps)]
    names = [k for k, _ in m.named_parameters()]

    def run(dtype, step):
        x = X.to(dtype, copy=True).requires_grad_(True)
        s0 = [s.to(dtype, copy=True).requires_grad_(True) for s in S0]
        state, outs = s0, []
        for t in range(steps):
            state = list(step(x[t], state))
            outs += state
        return x, s0, outs
    g = {}
    for dtype in (torch.float64, torch.float32):
        p = {k: v.detach().to(dtype, copy=True).requires_grad_(True) for k, v in m.named_parameters()}
        with _float64() if dtype == torch.float64 else contextlib.nullcontext():
            x, s0, o = run(dtype, lambda xt, st: lrgcn_cell(p, xt, ei, et, *st, R))
        g[dtype] = [torch.stack(o)] + _loss_grads(o, [w.to(dtype) for w in wgts], [x] + s0 + [p[k] for k in names])
    m.zero_grad(set_to_none=True)
    with _counted() as c:
        xf, sf, of = run(torch.float32, lambda xt, st: m(xt, ei, et, *st))
        gf = [torch.stack(of)] + _loss_grads(of, wgts, [xf] + sf + [p for _, p in m.named_parameters()])
    assert _ran(c) == {k: steps * v for k, v in _launches(R, co, True).items()}, c
    errs = []
    for label, got, r32, r64 in zip(["out", "dX", "dH0", "dC0"] + names, gf, g[torch.float32], g[torch.float64]):
        _check_err(errs, _family(R, co), got, r32, r64, (R, co, "recurrence", label))
    assert not errs, errs[:6]


@pytest.mark.parametrize("parts", PARTS)
@pytest.mark.parametrize("cin", [1, 10, 11, 16])
def test_wgrad2_reduce_is_the_fixed_order_sum(cin, parts):
    """stmp_lstm_rows_wgrad2: k_wide_rows_wgrad<2> (one partial per CTA of 32-row tiles for [dpi | dpf] and for [dpc | dpo]), then
    k_wide_rows_wgrad_reduce<2> into dw [128][nb] and db [128]; every element recomputed in float32 in the reduce's association
    (test_gpu_wgrad_reduce.py).  rows = 0 writes zeros."""
    torch.manual_seed(7 + cin)
    GCV = _lib.LSTM_GCONV
    nb, ld = ops.lstm_rows_nb(GCV, 2, cin), ops.lstm_rows_basis_ld(GCV, 2, cin)
    cap = 2 * _sms()
    rows = _rows(parts, 32, cap)
    n = _parts(rows, 32, cap)
    S, = _operands(rows, ld)
    dpre = _randn(2, max(rows, 1), 64)
    ws = _workspace(_lib.lib().stmp_lstm_rows_wgrad2_workspace_bytes(cin))
    dw = torch.full((128, nb), NAN, device=DEV)
    db = torch.full((128,), NAN, device=DEV)
    with _counted() as c:
        _check(_lib.lib().stmp_lstm_rows_wgrad2(cin, rows, ld, _lib.ptr(S), _lib.ptr(dpre), _lib.ptr(ws), _lib.ptr(dw), _lib.ptr(db),
                                                _lib.stream_ptr()))
    if rows == 0:
        assert not dw.any() and not db.any() and _ran(c) == {}
        return
    assert _ran(c) == {"k_lstm_rows_wgrad2": 1, "k_lstm_rows_wgrad2_reduce": 1}, c
    stride = ld * 64 + 64
    P = ws[:2 * n * stride].view(2, n, stride).cpu()
    row, col = torch.meshgrid(_ar(64), _ar(nb), indexing="ij")
    _equal(dw, torch.cat([_sum(P[g], col * 64 + row) for g in range(2)]))
    _equal(db, torch.cat([_sum(P[g], ld * 64 + _ar(64)) for g in range(2)]))


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
