"""The fused TGCN / A3TGCN kernels at 64 hidden channels (csrc/tgcn_attn.cu: k_tgcn_wide_attn<NQ, HAS_H>, k_tgcn_attn_bwd<NQ, 2> and
k_tgcn_wide_cell_bwd + the 64-wide weight-gradient contraction of rows.cuh), against float64 across their envelope and against the
op-for-op autograd path (`fused_training = False`), with the criterion of test_gpu_tgcn_envelope.py: the fused result's largest error
within 4x that of the same oracle in float32 plus 2^-20 of the tensor's scale."""
import contextlib

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN, A3TGCN2, TGCN, TGCN2
from test_gpu_graph_geometry import _counted, _float64
from test_gpu_tgcn_envelope import _at_offset, _check, _expect, _nq, _staged, make_graph
from tgcn64_seq import check_reference, data, load, model_for, oracle_run, run

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32 = torch.float64, torch.float32
W = 64
# tgcn_attn.cu: X[b] is staged up to these sizes; at 64 channels the forward with H keeps Bm (48.3 KB) next to it
FWD_STAGE_BYTES, BWD_STAGE_BYTES = 160 * 1024, 128 * 1024


def _model(cls, *args, flags=None, seed=0):
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
    """test_gpu_tgcn_envelope._reference at the module's width."""
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
            h = (torch.zeros(*x.shape[:nlead + 1], base.out_channels, device=DEV, dtype=dtype) if H is None
                 else pick(H).detach().to(dtype))
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


def _compare(m, X, ei, ew, H=None, wgt=None, grad_h=False, what=""):
    got, c = _fused(m, X, ei, ew, H, wgt, grad_h)
    _check(got, _reference(m, X, ei, ew, H, wgt, F32, grad_h), _reference(m, X, ei, ew, H, wgt, F64, grad_h), what)
    return c


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _close_grad(got, want):
    _close(got, want, 1e-3, 1e-3 * want.abs().max().item() + 1e-6)


# ==== 1. goldens from the unmodified reference (tests/golden/make_goldens_tgcn64.py) =====================================================
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", ["tgcn2_metr_la", "tgcn2_pems_bay", "tgcn_chickenpox", "a3tgcn2_cfg3", "a3tgcn_shared_h"])
def test_vs_reference_golden(golden_dir, name, fused):
    c = load(golden_dir)[name]
    d = data(c, DEV)
    outs, loss, grads, extra = oracle_run(c, d)
    check_reference(c, outs, loss, grads, extra)
    m = model_for(c, DEV, fused)
    with _counted() as cnt:
        got = run(m, c, d)
    wide = {"k_tgcn_wide_attn", "k_tgcn_wide_attn_bwd", "k_tgcn_wide_cell_bwd"}
    inference = c["kind"] == "a3_shared"                # fused_training only chooses the training path
    assert bool(wide & set(cnt)) == (fused or inference) and "k_tgcn_attn" not in cnt, cnt
    _close(got["out"], outs)
    if loss is not None:
        _close(got["loss"], loss, 1e-4, 1e-6)
        for k, g in grads.items():
            _close_grad(got["grads"][k], g)
        for k, g in extra.items():
            _close_grad(got[k], g)


# ==== 2. the float64 envelope ===========================================================================================================
GRAPHS = ([("random", n) for n in (1, 7, 64, 65, 325)]
          + [("hubs", 129), ("isolated", 65), ("improved", 64), ("selfloops", 63), ("dups", 129), ("unweighted", 325)])
WIDTHS = [(1, 1), (1, 33), (1, 65), (1, 128), (2, 12), (2, 64), (3, 11), (3, 42), (4, 8), (4, 32)]
CASES = list(dict.fromkeys([(*w, *GRAPHS[i % len(GRAPHS)]) for i, w in enumerate(WIDTHS)]
                           + [(*WIDTHS[i % len(WIDTHS)], *g) for i, g in enumerate(GRAPHS)]))


def test_every_nq_instance_is_exercised():
    assert {_nq(f, P) for f, P, _, _ in CASES} == {1, 2, 3, 4}
    assert {f for f, _, _, _ in CASES} == {1, 2, 3, 4} and max(f * P for f, P, _, _ in CASES) == 128
    assert {(k, n) for _, _, k, n in CASES} == set(GRAPHS)


@pytest.mark.parametrize("fin,P,kind,n", CASES, ids=[f"fin{f}-P{P}-{k}-N{n}" for f, P, k, n in CASES])
def test_a3tgcn64_vs_float64(fin, P, kind, n):
    ei, ew, flags = make_graph(kind, n)
    B = 3
    m = _model(A3TGCN2, fin, W, P, B, flags=flags, seed=fin * 1000 + P + n)
    gen = torch.Generator(device=DEV).manual_seed(fin * 1000 + P)
    X = torch.randn(B, n, fin, P, device=DEV, generator=gen)
    H = 0.5 * torch.randn(B, n, W, device=DEV, generator=gen)
    wgt = torch.randn(B, n, W, device=DEV, generator=gen)
    fg, bg = int(not _staged(FWD_STAGE_BYTES, X, n, fin * P)), int(not _staged(BWD_STAGE_BYTES, X, n, fin * P))
    for name, h in (("H=None", None), ("per-row H", H)):
        c = _compare(m, X, ei, ew, h, what=name)
        _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_attn[x-global]": fg, "k_tgcn_attn": 0, "k_spmm": 0})
    base = m._base_tgcn
    A, Bm, cc = base._packed3()
    with torch.no_grad(), _counted() as c:
        out = ops.tgcn_attn_fwd(base._plan(ei, ew, n), X, A, Bm, cc, torch.softmax(m._attention, 0), H[0], h_shared=True)
    _expect(c, {"k_tgcn_wide_attn": 1})
    Hs = H[:1].expand(B, n, W)
    _check({"out": out}, _reference(m, X, ei, ew, Hs, None, F32), _reference(m, X, ei, ew, Hs, None, F64), "shared H")
    got, c = _fused(m, X, ei, ew, None, wgt)
    _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_attn_bwd": 1, "k_tgcn_wide_attn_bwd_reduce": 1, "k_tgcn_wide_attn[x-global]": fg,
                "k_tgcn_wide_attn_bwd[x-global]": bg, "k_tgcn_attn_bwd": 0, "k_spmm": 0})
    _check(got, _reference(m, X, ei, ew, None, wgt, F32), _reference(m, X, ei, ew, None, wgt, F64), "training")


CELL_GRAPHS = [("hubs", 129), ("isolated", 65), ("improved", 64), ("selfloops", 63), ("dups", 129), ("unweighted", 325), ("random", 1),
               ("random", 7)]
CELL_LAUNCHES = ("k_tgcn_wide_cell_bwd", "k_tgcn_wide_wgrad", "k_tgcn_wide_wgrad_reduce", "k_tgcn_wide_wgrad_unpack")


@pytest.mark.parametrize("cls", [TGCN, TGCN2])
@pytest.mark.parametrize("fin", [1, 2, 3, 4])
def test_tgcn64_cell_training_vs_float64(cls, fin):
    i = 2 * fin + (cls is TGCN2)
    for kind, n in (CELL_GRAPHS[i % 8], CELL_GRAPHS[(i + 3) % 8]):
        ei, ew, flags = make_graph(kind, n)
        m = _model(cls, *((fin, W) if cls is TGCN else (fin, W, 3)), flags=flags, seed=i + n)
        lead = () if cls is TGCN else (3,)
        gen = torch.Generator(device=DEV).manual_seed(i)
        X0, X1 = (torch.randn(*lead, n, fin, device=DEV, generator=gen) for _ in range(2))
        H = 0.5 * torch.randn(*lead, n, W, device=DEV, generator=gen)
        wgt = torch.randn(*lead, n, W, device=DEV, generator=gen)
        fg, bg = int(not _staged(FWD_STAGE_BYTES, X0, n, fin)), int(not _staged(BWD_STAGE_BYTES, X0, n, fin))
        c = _compare(m, X0, ei, ew, None, wgt, what=(kind, n, "first step"))
        _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_attn_bwd": 1, "k_tgcn_wide_cell_bwd": 0, "k_tgcn_wide_attn_bwd[x-global]": bg})
        c = _compare(m, X1, ei, ew, H, wgt, grad_h=True, what=(kind, n, "carried state"))
        _expect(c, {"k_tgcn_wide_attn": 1, **{k: 1 for k in CELL_LAUNCHES}, "k_tgcn_wide_attn_bwd": 0, "k_tgcn_cell_bwd": 0,
                    "k_tgcn_wide_attn[x-global]": fg, "k_tgcn_wide_cell_bwd[x-global]": bg})
        c = _compare(m, X1, ei, ew, H, what=(kind, n, "inference with H"))
        _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_attn[x-global]": fg})


# ---- staging limits: both sides of each, with H (Bm staged next to X) and without, and a misaligned X ---------------------------------
ROW = 4 * 4 * 32                                       # bytes of a node's row at fin = 4, P = 32
STAGING = [  # (fin, P, N, x at a 4-byte offset, forward staged, backward staged)
    (4, 32, BWD_STAGE_BYTES // ROW, False, True, True),
    (4, 32, BWD_STAGE_BYTES // ROW + 1, False, True, False),
    (4, 32, FWD_STAGE_BYTES // ROW, False, True, False),
    (4, 32, FWD_STAGE_BYTES // ROW + 1, False, False, False),
    (2, 12, 64, True, False, False),
]


@pytest.mark.parametrize("fin,P,n,offset,fwd_staged,bwd_staged", STAGING,
                         ids=[f"fin{f}-P{P}-N{n}" + ("-offset4" if o else "") for f, P, n, o, _, _ in STAGING])
def test_staging_limits(fin, P, n, offset, fwd_staged, bwd_staged):
    ei, ew, flags = make_graph("random", n)
    B = 2
    m = _model(A3TGCN2, fin, W, P, B, flags=flags, seed=n)
    gen = torch.Generator(device=DEV).manual_seed(n)
    X = torch.randn(B, n, fin, P, device=DEV, generator=gen)
    H = 0.5 * torch.randn(B, n, W, device=DEV, generator=gen)
    wgt = torch.randn(B, n, W, device=DEV, generator=gen)
    if offset:
        X = _at_offset(X)
    assert _staged(FWD_STAGE_BYTES, X, n, fin * P) == fwd_staged and _staged(BWD_STAGE_BYTES, X, n, fin * P) == bwd_staged
    for h in (None, H):
        c = _compare(m, X, ei, ew, h, what="inference")
        _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_attn[x-global]": int(not fwd_staged)})
    c = _compare(m, X, ei, ew, None, wgt, what="training")
    _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_attn_bwd": 1, "k_tgcn_wide_attn[x-global]": int(not fwd_staged),
                "k_tgcn_wide_attn_bwd[x-global]": int(not bwd_staged)})
    if offset:                                         # the cell backward gathers from global memory as well
        mc = _model(TGCN2, fin, W, B, seed=n)
        Xc = _at_offset(torch.randn(B, n, fin, device=DEV, generator=gen))
        c = _compare(mc, Xc, ei, ew, H, wgt, grad_h=True, what="cell")
        _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_cell_bwd": 1, "k_tgcn_wide_attn[x-global]": 1, "k_tgcn_wide_cell_bwd[x-global]": 1})


@pytest.mark.parametrize("extra", [0, 1])
def test_cell_backward_staging_limit(extra):
    fin, B = 4, 2
    n = BWD_STAGE_BYTES // (4 * fin) + extra
    ei, ew, flags = make_graph("random", n)
    m = _model(TGCN2, fin, W, B, flags=flags, seed=extra)
    gen = torch.Generator(device=DEV).manual_seed(n)
    X = torch.randn(B, n, fin, device=DEV, generator=gen)
    H = 0.5 * torch.randn(B, n, W, device=DEV, generator=gen)
    wgt = torch.randn(B, n, W, device=DEV, generator=gen)
    assert _staged(FWD_STAGE_BYTES, X, n, fin) and _staged(BWD_STAGE_BYTES, X, n, fin) == (extra == 0)
    c = _compare(m, X, ei, ew, H, wgt, grad_h=True)
    _expect(c, {"k_tgcn_wide_attn": 1, "k_tgcn_wide_cell_bwd": 1, "k_tgcn_wide_attn[x-global]": 0, "k_tgcn_wide_cell_bwd[x-global]": extra})


def test_50k_node_graph():
    """X[b] of 50 000 nodes x 4 features is 800 KB: every kernel gathers from global memory."""
    ei, ew = synthetic.large_graph(50000, 200000, seed=3)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    m = _model(TGCN2, 4, W, 2, seed=2)
    gen = torch.Generator(device=DEV).manual_seed(2)
    X0, X1 = (torch.randn(2, 50000, 4, device=DEV, generator=gen) for _ in range(2))
    H = 0.5 * torch.randn(2, 50000, W, device=DEV, generator=gen)
    wgt = torch.randn(2, 50000, W, device=DEV, generator=gen)
    c = _compare(m, X0, ei, ew, None, wgt, what="first step")
    _expect(c, {"k_tgcn_wide_attn[x-global]": 1, "k_tgcn_wide_attn_bwd[x-global]": 1})
    c = _compare(m, X1, ei, ew, H, wgt, grad_h=True, what="carried state")
    _expect(c, {"k_tgcn_wide_attn[x-global]": 1, "k_tgcn_wide_cell_bwd[x-global]": 1, "k_tgcn_wide_wgrad": 1})


# ---- batch rows -------------------------------------------------------------------------------------------------------------------------
def _row_models(B, n, flags):
    return _model(A3TGCN2, 1, W, 2, B, flags=flags, seed=B), _model(TGCN2, 1, W, B, flags=flags, seed=B + 1)


def test_one_batch_row():
    ei, ew, flags = make_graph("hubs", 129)
    ma, mc = _row_models(1, 129, flags)
    gen = torch.Generator(device=DEV).manual_seed(1)
    X = torch.randn(1, 129, 1, 2, device=DEV, generator=gen)
    H = 0.5 * torch.randn(1, 129, W, device=DEV, generator=gen)
    wgt = torch.randn(1, 129, W, device=DEV, generator=gen)
    _expect(_compare(ma, X, ei, ew, H), {"k_tgcn_wide_attn": 1})
    _expect(_compare(ma, X, ei, ew, None, wgt), {"k_tgcn_wide_attn": 1, "k_tgcn_wide_attn_bwd": 1})
    _expect(_compare(mc, X[..., 0], ei, ew, H, wgt, grad_h=True), {"k_tgcn_wide_attn": 1, "k_tgcn_wide_cell_bwd": 1})


@pytest.mark.parametrize("B,fused", [(65535, True), (65536, False)])
def test_largest_batches(B, fused):
    n = 7
    ei, ew, flags = make_graph("random", n)
    ma, mc = _row_models(B, n, flags)
    gen = torch.Generator(device=DEV).manual_seed(7)
    X = torch.randn(B, n, 1, 2, device=DEV, generator=gen)
    H = 0.5 * torch.randn(B, n, W, device=DEV, generator=gen)
    wgt = torch.randn(B, n, W, device=DEV, generator=gen)
    try:
        _expect(_compare(ma, X, ei, ew, H, what="A3TGCN2 with H"), {"k_tgcn_wide_attn": int(fused)})
        # The attention gradient sums g * H_t over 65 535 x 7 x 64 products per period, and the softmax backward then cancels most of it.
        # The fused one was measured at 9.0e-5 from float64 against the fp32 oracle's 4.5e-6, at scale 19; 8x the fp32 error plus
        # 2^-20 of the scale allows 5.4e-5.  That is the open point of test_gpu_tgcn_envelope._check, at twice the channels: the gates'
        # __expf / __fdividef errors add up as a random walk over the products.  The attention gradient is held to 32x here and every
        # other tensor to the usual criterion.
        got, c = _fused(ma, X, ei, ew, None, wgt)
        _expect(c, {"k_tgcn_wide_attn": int(fused), "k_tgcn_wide_attn_bwd": int(fused)})
        r32, r64 = _reference(ma, X, ei, ew, None, wgt, F32), _reference(ma, X, ei, ew, None, wgt, F64)
        _check({k: v for k, v in got.items() if k != "_attention"}, r32, {k: v for k, v in r64.items() if k != "_attention"}, "training")
        e = float((got["_attention"].double() - r64["_attention"]).abs().max())
        e32 = float((r32["_attention"].double() - r64["_attention"]).abs().max())
        assert e <= 32 * e32 + 2.0 ** -20 * float(r64["_attention"].abs().max()), (e, e32)
        _expect(_compare(mc, X[..., 0], ei, ew, H, wgt, grad_h=True, what="TGCN2 carried state"),
                {"k_tgcn_wide_attn": int(fused), "k_tgcn_wide_cell_bwd": int(fused)})
    finally:
        del X, H, wgt
        torch.cuda.empty_cache()


def test_empty_batch_training():
    ei, ew, flags = make_graph("random", 65)
    ma, mc = _row_models(0, 65, flags)
    for m, X, H in ((ma, torch.randn(0, 65, 1, 2, device=DEV), None), (mc, torch.randn(0, 65, 1, device=DEV), None),
                    (mc, torch.randn(0, 65, 1, device=DEV), torch.randn(0, 65, W, device=DEV))):
        got, c = _fused(m, X, ei, ew, H, torch.randn(0, 65, W, device=DEV), grad_h=H is not None)
        assert got["out"].shape == (0, 65, W)
        for k, g in got.items():
            assert g is not None and not bool(g.any()), k
        assert not any(k.startswith("k_tgcn") for k in c), c


# ==== 3. fused cell backward against autograd, bit-equality and determinism ===============================================================
def _graph(seed=0):
    ei, ew, _ = synthetic.metr_la_like(seed, 16)
    return torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)


def _cell_case(cls, fin, improved=False, add_self_loops=True, B=3, seed=0):
    m = _model(cls, *((fin, W) if cls is TGCN else (fin, W, B)), flags=dict(improved=improved, add_self_loops=add_self_loops), seed=seed)
    lead = () if cls is TGCN else (B,)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(*lead, 207, fin, device=DEV, generator=gen)
    H = torch.randn(*lead, 207, W, device=DEV, generator=gen) * 0.5
    w = torch.randn(*lead, 207, W, device=DEV, generator=gen)
    return m, X, H, w


@pytest.mark.parametrize("cls", [TGCN, TGCN2])
@pytest.mark.parametrize("fin", [1, 2, 3, 4])
def test_fused_cell_backward_vs_autograd(cls, fin):
    ei, ew = _graph(1)
    for improved in (False, True):
        for add_self_loops in (True, False):
            for h_grad in (True, False):
                m, X, H, w = _cell_case(cls, fin, improved, add_self_loops)
                res = []
                for fused in (True, False):
                    m.fused_training = fused
                    m.zero_grad(set_to_none=True)
                    Hl = H.clone().requires_grad_(h_grad)
                    with _counted() as c:
                        out = m(X, ei, ew, Hl)
                        (out * w).sum().backward()
                    assert c.get("k_tgcn_wide_cell_bwd", 0) == int(fused)
                    res.append((out.detach(), Hl.grad, {k: p.grad.clone() for k, p in m.named_parameters()}))
                (of, hf, gf), (oa, ha, ga) = res
                _close(of, oa)
                assert (hf is None) == (not h_grad)
                if h_grad:
                    _close_grad(hf, ha)
                for k in ga:
                    _close_grad(gf[k], ga[k])


def test_training_forward_is_bit_equal_to_inference():
    ei, ew = _graph()
    m, X, H, _ = _cell_case(TGCN2, 2)
    for h in (None, H):
        with _counted() as c:
            out = m(X, ei, ew, h)
        assert out.requires_grad and c.get("k_tgcn_wide_attn", 0) == 1
        with torch.no_grad():
            ref = m(X, ei, ew, h)
        assert torch.equal(out.detach(), ref)
    a = _model(A3TGCN2, 2, W, 12, 3, seed=1)
    X12 = torch.randn(3, 207, 2, 12, device=DEV)
    out = a(X12, ei, ew)
    with torch.no_grad():
        assert torch.equal(out.detach(), a(X12, ei, ew))


def test_backward_is_deterministic():
    ei, ew = _graph()
    m, X, H, w = _cell_case(TGCN2, 4, B=16)
    a = _model(A3TGCN2, 2, W, 64, 4, seed=5)
    X64 = torch.randn(4, 207, 2, 64, device=DEV)
    w64 = torch.randn(4, 207, W, device=DEV)

    def grads():
        m.zero_grad(set_to_none=True)
        a.zero_grad(set_to_none=True)
        Hl = H.clone().requires_grad_(True)
        (m(X, ei, ew, Hl) * w).sum().backward()
        (m(X, ei, ew) * w).sum().backward()
        (a(X64, ei, ew) * w64).sum().backward()
        return [Hl.grad] + [p.grad.clone() for p in m.parameters()] + [p.grad.clone() for p in a.parameters()]
    for x, y in zip(grads(), grads()):
        assert torch.equal(x, y)


# ==== 4. launches, CUDA graphs, routing and the ABI ========================================================================================
def test_launches_of_a_batched_tgcn_training_step(golden_dir):
    """A 12-step BatchedTGCN step at 64 channels: 12 forwards, one H = None backward (2 launches) and 11 cell backwards (4 launches each),
    no SpMM and nothing else from the library."""
    c = load(golden_dir)["tgcn2_metr_la"]
    m, d = model_for(c, DEV, True), data(c, DEV)
    run(m, c, d)                                       # plans and folded weights
    n0 = _lib.launch_count()
    with _counted() as cnt:
        run(m, c, d)
    torch.cuda.synchronize()
    want = {"k_tgcn_wide_attn": 12, "k_tgcn_wide_attn_bwd": 1, "k_tgcn_wide_attn_bwd_reduce": 1, **{k: 11 for k in CELL_LAUNCHES},
            "k_spmm": 0, "k_tgcn_attn": 0}
    _expect(cnt, want)
    assert _lib.launch_count() - n0 == 12 + 2 + 4 * 11


def test_cuda_graph_replay_of_a_training_step(golden_dir):
    c = load(golden_dir)["tgcn2_pems_bay"]
    m = model_for(c, DEV, True)
    d = data(c, DEV)                                   # no host-to-device copy inside the capture
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)
    state0 = {k: v.clone() for k, v in m.state_dict().items()}

    def step(model, o):
        o.zero_grad(set_to_none=False)
        loss = run(model, c, d, backward=False)["loss"]
        loss.backward()
        o.step()
        return loss

    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step(m, opt)
    torch.cuda.current_stream().wait_stream(side)
    m_e = model_for(c, DEV, True)
    m_e.load_state_dict(state0)
    opt_e = torch.optim.Adam(m_e.parameters(), lr=1e-3)
    eager = [step(m_e, opt_e).detach() for _ in range(2)]
    m.load_state_dict(state0)
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step(m, opt)
    m.load_state_dict(state0)
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    replay = []
    for _ in range(2):
        graph.replay()
        replay.append(loss.detach().clone())
    torch.cuda.synchronize()
    for a, b in zip(replay, eager):
        _close(a, b, 1e-5, 1e-7)
    for p, pe in zip(m.parameters(), m_e.parameters()):
        _close(p, pe, 1e-5, 1e-6)


def test_routing():
    ei, ew = _graph()
    gen = torch.Generator(device=DEV).manual_seed(3)
    X = torch.randn(3, 207, 2, device=DEV, generator=gen)
    H = 0.5 * torch.randn(3, 207, W, device=DEV, generator=gen)
    with _counted() as c:
        Xg = X.clone().requires_grad_(True)
        _model(TGCN2, 2, W, 3)(Xg, ei, ew, H).sum().backward()                                      # gradient w.r.t. X
        _model(TGCN2, 5, W, 3)(torch.randn(3, 207, 5, device=DEV), ei, ew, H).sum().backward()      # in_channels 5
        with torch.no_grad():
            _model(TGCN2, 5, W, 3)(torch.randn(3, 207, 5, device=DEV), ei, ew, H)
        _model(A3TGCN2, 2, W, 65, 3)(torch.randn(3, 207, 2, 65, device=DEV), ei, ew).sum().backward()   # in_channels * periods 130
        Hg = H.clone().requires_grad_(True)
        _model(A3TGCN2, 2, W, 4, 3)(torch.randn(3, 207, 2, 4, device=DEV), ei, ew, Hg).sum().backward()  # A3TGCN with a state to train
        _model(TGCN2, 2, 48, 3)(X, ei, ew, H[..., :48]).sum().backward()                           # out_channels 48
        with torch.no_grad():
            _model(TGCN2, 2, 48, 3)(X, ei, ew, H[..., :48])
    assert Xg.grad is not None and Hg.grad is not None
    assert not any(k.startswith("k_tgcn") for k in c) and c.get("k_spmm", 0) > 0, c
    # the 32-wide routes are unchanged: the 32-wide kernels and no 64-wide one
    m32 = _model(TGCN2, 2, 32, 3)
    with _counted() as c:
        m32(X, ei, ew).sum().backward()
        m32(X, ei, ew, H[..., :32]).sum().backward()
        with torch.no_grad():
            m32(X, ei, ew, H[..., :32])
        _model(A3TGCN2, 2, 32, 12, 3)(torch.randn(3, 207, 2, 12, device=DEV), ei, ew).sum().backward()
    _expect(c, {"k_tgcn_attn": 4, "k_tgcn_attn_bwd": 2, "k_tgcn_cell_bwd": 1, "k_tgcn_wide_attn": 0, "k_tgcn_wide_attn_bwd": 0,
                "k_tgcn_wide_cell_bwd": 0})


def test_abi_errors():
    ei, ew = _graph()
    m = TGCN2(2, W, 1).to(DEV)
    plan = m._plan(ei, ew, 207)
    L = _lib.lib()
    buf = torch.zeros(1 << 20, device=DEV)
    p, st = _lib.ptr(buf), _lib.stream_ptr()
    cell = lambda B, fin, x: (plan.handle, B, fin, x, p, 207 * W, p, p, p, p, p, p, p, p, p, st)
    assert L.stmp_tgcn_wide_cell_bwd(*cell(1, 5, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_wide_cell_bwd(*cell(1, 0, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_wide_cell_bwd(*cell(1, 2, None)) == _lib.STMP_EINVAL
    assert L.stmp_tgcn_wide_cell_bwd(*cell(65536, 2, p)) == _lib.STMP_ESHAPE
    assert L.stmp_tgcn_wide_cell_bwd(None, *cell(1, 2, p)[1:]) == _lib.STMP_EINVAL
    fwd = lambda B, fin, x: (plan.handle, B, fin, 1, x, None, 0, p, p, p, None, p, st)
    assert L.stmp_tgcn_wide_attn_fwd(*fwd(1, 5, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_wide_attn_fwd(*fwd(1, 0, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_wide_attn_fwd(*fwd(1, 2, None)) == _lib.STMP_EINVAL
    assert L.stmp_tgcn_wide_attn_fwd(*fwd(65536, 2, p)) == _lib.STMP_ESHAPE
    assert L.stmp_tgcn_wide_attn_fwd(None, *fwd(1, 2, p)[1:]) == _lib.STMP_EINVAL
    bwd = lambda B, fin, x: (plan.handle, B, fin, 1, x, p, p, None, p, p, p, p, None, st)
    assert L.stmp_tgcn_wide_attn_bwd(*bwd(1, 5, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_wide_attn_bwd(*bwd(1, 0, p)) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_tgcn_wide_attn_bwd(*bwd(1, 2, None)) == _lib.STMP_EINVAL
    assert L.stmp_tgcn_wide_attn_bwd(*bwd(65536, 2, p)) == _lib.STMP_ESHAPE
    assert L.stmp_tgcn_wide_attn_bwd(None, *bwd(1, 2, p)[1:]) == _lib.STMP_EINVAL
    assert L.stmp_tgcn_wide_attn_bwd_workspace_bytes(plan.handle, 2) == 2 * 4 * (10 * 64 + 128) * 4     # 207 nodes: 4 CTAs per row
    assert L.stmp_tgcn_wide_cell_bwd_workspace_bytes(plan.handle, 2) > 2 * 207 * (192 + 2 * 72) * 4
    torch.cuda.synchronize()
