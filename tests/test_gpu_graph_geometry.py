"""The one-SM fused recurrence kernels on adversarial graphs: the compact graph formats they read, checked structurally and through
the kernels against float64.

Every kernel that keeps a whole graph on one SM reads it from a compact format the plan builds:
  * the wgmma forward reads two images.  The CTA-pair kernel `k_dcrnn_seq_tc` (small batches, the `[cluster2]` counter) reads the
    shared-memory graph image (csrc/graph_image.cuh) -- 8-bit rows, pad entries that point at zero row 207, edges in groups of four
    with a 7-bit group count per task, tasks cut into segments by 128-row tile and operator and dealt to 16 warps longest-first.
    Windows not served by a CTA pair (the B = 200 cases here) run the one-CTA kernel `k_dcrnn_seq_rf`, which gathers straight into
    wgmma register fragments from the row image (csrc/row_image.cuh).  Each image exists only if it fits its kernel's shared memory,
    and the wgmma path takes a plan only when it has both (`tc_fits`).  This file decodes the graph image only; the
    `ops.gru_seq_supported(...) == image_fits(...)` assertions below therefore hold because on these graphs the row image is never
    the tighter limit, and the B = 200 cases check the row-image kernel numerically;
  * the persistent backward (csrc/dcrnn_bwd.cu) reads the transposed operators from a compressed shared-memory copy when it fits
    beside the per-window buffers (`graph_in_smem`), otherwise from the global CSR (path counter `k_*_bwd_seq[graph-global]`);
  * the FFMA forward `k_dcrnn_seq` picks one of five row mappings by N.
A dropped edge or a mis-sorted task can stay numerically invisible on a random graph, so the image is decoded and checked against the
plan's CSR (`stmp_plan_export`) as well as run.

Numerical criterion (the idiom of test_gpu_split_precision.py): against the float64 oracle (`oracle.recurrent`, run in float64 on the
GPU), the fused path's largest error must stay within 4x that of the fp32 op-for-op path plus 2^-20 of the tensor's scale.  The
graphs: random sparse graphs at N around the 64-row subtile and 128-row tile boundaries, hubs, rows of every degree residue mod 4, a
last row with nothing but a self loop, a ring, the densest graph that still gets an image (and 4 edges more), and graphs either side of
the backward's staged-copy limit at 104 and 112 basis columns.  Every node has in- and out-degree >= 1, so DConv stays finite."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN, GConvGRU
from pytorch_geometric_temporal_b200.nn.recurrent.dcrnn import _DcrnnSeqFn
from pytorch_geometric_temporal_b200.plan import GraphPlan

pytestmark = pytest.mark.gpu
DEV = "cuda"

# ---- the formats' constants and size formulas (graph_image.cuh, plan.cu, dcrnn_seq_tc.cu tc_layout, dcrnn_bwd.cu) ------------------
IMG_MAX_N, ZERO_ROW, NO_TASK, WARPS, SEGS = 207, 207, 0xFFFFFFFF, 16, 4
LPT_A, LPT_B, LPT_HANDICAP = 2, 3, 24
TC_SMEM = 232448
TC_FIXED = 4 * 208 * 128 + 4 * 96 * 128 + 208 * 36 * 4 + 96 * 4 + 8     # A panels, B panels, gather buffer U, biases, mbarrier
BWD_SMEM = 227 * 1024 - 16                                            # less the CTA pair's static mbarrier


def _a16(v):
    return (v + 15) & ~15


def image_layout(n_tasks, nnz):
    cap_wt = (n_tasks + 3) // 4 + SEGS
    cap_groups = (nnz + 3 * n_tasks) // 4 + 2
    off_wstart, off_wcount = 16, 16 + WARPS * SEGS * 2
    off_wt = _a16(off_wcount + WARPS * SEGS * 2)
    off_idx = off_wt + _a16(cap_wt * 16)
    off_val = off_idx + _a16(cap_groups * 4)
    return dict(wstart=off_wstart, wcount=off_wcount, wt=off_wt, idx=off_idx, val=off_val, bytes=_a16(off_val + cap_groups * 16))


def image_fits(n, n_ops, nnz):
    return n <= IMG_MAX_N and image_layout(n_ops * n, nnz)["bytes"] <= TC_SMEM - TC_FIXED


def ncol_of(cin, nops=2):
    return ((nops + 1) * (cin + 32) + 7) // 8 * 8


def bwd_staged(n, cin, nnz_per_op):
    """graph_in_smem: does the persistent backward stage the transposed operators in shared memory?"""
    nops = len(nnz_per_op)
    if nops == 0 or any(z >= 65536 for z in nnz_per_op) or n > 256:
        return False
    ncol, rg = ncol_of(cin, nops), (n + 7) // 8
    base = 4 * (3 * 32 * ncol + rg * 8 * ncol + 2 * 32 * (rg * 8 + 4) + n * 36)
    nnz = sum(nnz_per_op)
    return base + 4 * nnz + ((nnz + 3) & ~3) + 2 * nops * (n + 1) + 8 <= BWD_SMEM


def densest_image_edges(n):
    """Largest edge count E whose DConv plan (2E entries over two operators) still has an image at N = n."""
    e = 0
    while image_fits(n, 2, 2 * (e + 1)):
        e += 1
    return e


def staged_limit_edges(n, cin):
    e = 0
    while bwd_staged(n, cin, [e + 1, e + 1]):
        e += 1
    return e


# ---- the graph family -----------------------------------------------------------------------------------------------------------------
def _unique(src, dst):
    key = src.astype(np.int64) * 100_000 + dst
    _, first = np.unique(key, return_index=True)
    keep = np.sort(first)
    return src[keep], dst[keep]


def make_graph(kind, n, edges=None, seed=0):
    """(src, dst, weight) as numpy arrays; every node has in- and out-degree >= 1, no duplicate edges."""
    rng = np.random.default_rng([seed, n, sum(map(ord, kind))])
    ring = np.arange(n)
    src, dst = ring, (ring + 1) % n
    if kind == "random":
        src = np.concatenate([src, rng.integers(0, n, 3 * n)])
        dst = np.concatenate([dst, rng.integers(0, n, 3 * n)])
    elif kind == "hubs":                                   # in-hub: N - 1 edges into the last row; out-hub: N - 1 edges out of row 3
        others_in, others_out = np.delete(ring, n - 1), np.delete(ring, 3)
        src = np.concatenate([src, rng.integers(0, n, 2 * n), others_in, np.full(n - 1, 3)])
        dst = np.concatenate([dst, rng.integers(0, n, 2 * n), np.full(n - 1, n - 1), others_out])
    elif kind == "mod4":                                   # in-degree of row i = 1 + i % 9: every residue mod 4, short and long
        extra_s, extra_d = [], []
        for i in range(n):
            cand = rng.permutation(np.delete(ring, [i, (i - 1) % n]))[: i % 9]
            extra_s.append(cand)
            extra_d.append(np.full(cand.size, i))
        src, dst = np.concatenate([src] + extra_s), np.concatenate([dst] + extra_d)
    elif kind == "lonely":                                 # the last row has nothing but a self loop
        m = n - 1
        r = np.arange(m)
        src = np.concatenate([r, rng.integers(0, m, 3 * m), [m]])
        dst = np.concatenate([(r + 1) % m, rng.integers(0, m, 3 * m), [m]])
    elif kind == "edges":                                  # exactly `edges` edges: the ring plus random distinct pairs
        taken = set((src * n + dst).tolist())
        perm = [p for p in rng.permutation(n * n).tolist() if p not in taken][: edges - n]
        perm = np.array(perm, dtype=np.int64)
        src, dst = np.concatenate([src, perm // n]), np.concatenate([dst, perm % n])
    else:
        assert kind == "ring"
    src, dst = _unique(src.astype(np.int64), dst.astype(np.int64))
    if kind == "edges":
        assert src.size == edges
    w = (rng.random(src.size) + 0.1).astype(np.float32)
    return src, dst, w


def _tensors(g):
    src, dst, w = g
    return torch.from_numpy(np.stack([src, dst])).to(DEV), torch.from_numpy(w).to(DEV)


E_DENSE = densest_image_edges(207)
E_104, E_112 = staged_limit_edges(207, 2), staged_limit_edges(207, 3)
GEOMETRIES = ([("random", n, None) for n in (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 206, 207)]
              + [(k, n, None) for n in (129, 207) for k in ("hubs", "mod4", "lonely", "ring")]
              + [("edges", 207, E_DENSE), ("edges", 207, E_DENSE + 4)]
              + [("edges", 207, e) for e in (E_104, E_104 + 1, E_112, E_112 + 1)])
GEO_IDS = [f"{k}-N{n}" + (f"-E{e}" if e else "") for k, n, e in GEOMETRIES]


@contextlib.contextmanager
def _counted():
    """Yields a dict that, after the block, holds {kernel: launches during the block}."""
    c0, delta = _lib.path_counters(), {}
    yield delta
    c1 = _lib.path_counters()
    delta.update({k: v - c0.get(k, 0) for k, v in c1.items() if v != c0.get(k, 0)})


@contextlib.contextmanager
def _option(name, value, default):
    _lib.set_option(name, value)
    try:
        yield
    finally:
        _lib.set_option(name, default)


@contextlib.contextmanager
def _float64():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)       # the oracle's zeros / ones / scatter buffers
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def _assert_err(got, ref32, ref64, what):
    got, ref32 = got.detach().double(), ref32.detach().double()
    assert bool(torch.isfinite(got).all()), what
    e, e32 = float((got - ref64).abs().max()), float((ref32 - ref64).abs().max())
    scale = float(ref64.abs().max())
    assert e <= 4 * e32 + 2.0 ** -20 * scale, (what, "fused / fp32 op-for-op error vs float64", e, e32, scale)


# ==== 1. the graph image, decoded ========================================================================================================
def _decode(img, n, n_ops, nnz):
    L = image_layout(n_ops * n, nnz)
    a = img.numpy()
    assert a.size == L["bytes"]
    hdr = a[:16].view(np.int32)
    nwt, ngr = int(hdr[0]), int(hdr[1])
    return dict(hdr=hdr, nwt=nwt, ngroups=ngr,
                wstart=a[L["wstart"]:L["wstart"] + 128].view(np.uint16).reshape(WARPS, SEGS).astype(np.int64),
                wcount=a[L["wcount"]:L["wcount"] + 128].view(np.uint16).reshape(WARPS, SEGS).astype(np.int64),
                wt=a[L["wt"]:L["wt"] + 16 * nwt].view(np.uint32).reshape(nwt, 4),
                idx=a[L["idx"]:L["idx"] + 4 * (ngr + 1)].view(np.uint32),
                val=a[L["val"]:L["val"] + 16 * (ngr + 1)].view(np.uint32).reshape(ngr + 1, 4))


def check_image(plan, n_ops):
    """Decodes the plan's image for n_ops operators and checks it against the plan's CSR."""
    n = plan.num_nodes
    csr = []
    for op in range(n_ops):
        rp, col, val, _ = plan.export(op)
        csr.append((rp.cpu().numpy(), col.cpu().numpy(), val.cpu().view(torch.int32).numpy().view(np.uint32)))
    nnz = sum(int(c[0][-1]) for c in csr)
    img = plan.graph_image(n_ops)
    assert img is not None
    im = _decode(img, n, n_ops, nnz)
    deg = np.concatenate([np.diff(c[0]) for c in csr])                       # task id = op * N + row
    ng = (deg + 3) // 4
    g0 = np.concatenate([[0], np.cumsum(ng)])
    seg_of_task = 2 * (np.tile(np.arange(n), n_ops) >= 128) + np.repeat(np.arange(n_ops), n)
    seg_cnt = np.bincount(seg_of_task, minlength=SEGS)
    # header
    assert im["hdr"][2] == 1 and im["hdr"][3] == 0
    assert im["ngroups"] == int(ng.sum())
    assert im["nwt"] == int(((seg_cnt + 3) // 4).sum())
    # warp ranges: disjoint, cover every warp-task, segments in order
    slot_seg, slot_warp, nxt = np.full(im["nwt"], -1), np.full(im["nwt"], -1), 0
    for s in range(SEGS):
        for w in range(WARPS):
            st, c = int(im["wstart"][w, s]), int(im["wcount"][w, s])
            assert st == nxt, ("warp ranges are not contiguous in (segment, warp) order", s, w, st, nxt)
            slot_seg[st:st + c], slot_warp[st:st + c] = s, w
            nxt += c
    assert nxt == im["nwt"]
    # tasks: each (row, op) once, in its segment, with its group count and first group
    seen = np.zeros(n_ops * n, dtype=np.int64)
    seg_wts = [[] for _ in range(SEGS)]
    for slot in range(im["nwt"]):
        d = im["wt"][slot].astype(np.int64)
        tasks = []
        for q in range(4):
            if d[q] == NO_TASK:
                tasks.append(None)
                continue
            row, op, g, first = d[q] & 0xFF, (d[q] >> 8) & 1, (d[q] >> 9) & 0x7F, d[q] >> 16
            assert op < n_ops and row < n
            task = op * n + row
            seen[task] += 1
            assert seg_of_task[task] == slot_seg[slot], ("task in the wrong segment", row, op, slot_seg[slot])
            assert g == ng[task] and first == g0[task], ("task descriptor", row, op, g, ng[task], first, g0[task])
            tasks.append(task)
        seg_wts[slot_seg[slot]].append((slot, tasks))
    assert (seen == 1).all(), ("tasks missing or repeated", np.nonzero(seen != 1)[0][:8])
    # rank order inside a segment: (group count desc, task id asc) over the warp-tasks' quarters; only the last warp-task has holes
    for s in range(SEGS):
        wts = seg_wts[s]
        assert len(wts) == (seg_cnt[s] + 3) // 4
        order = sorted(wts, key=lambda st: (-ng[st[1][0]], st[1][0]))
        flat = [t for _, ts in order for t in ts]
        real = [t for t in flat if t is not None]
        assert flat[:len(real)] == real, ("empty quarters before the segment's last warp-task", s)
        assert len(flat) - len(real) == 4 * len(wts) - seg_cnt[s]
        keys = [(-ng[t], t) for t in real]
        assert keys == sorted(keys), ("tasks of a segment out of rank order", s)
        for w in range(WARPS):                           # a warp runs its warp-tasks in rank order
            mine = [ts[0] for slot, ts in wts if slot_warp[slot] == w]
            assert [(-ng[t], t) for t in mine] == sorted((-ng[t], t) for t in mine)
    # edges: each task's groups are its CSR row in CSR order, values bit for bit; pads are (207, +0.0); one all-pad spare group
    rows = ((im["idx"][:, None] >> np.array([0, 8, 16, 24], dtype=np.uint32)) & 0xFF).astype(np.int64)
    for task in range(n_ops * n):
        op, i = divmod(task, n)
        rp, col, valb = csr[op]
        b, e = int(rp[i]), int(rp[i + 1])
        got_r = rows[g0[task]:g0[task + 1]].reshape(-1)
        got_v = im["val"][g0[task]:g0[task + 1]].reshape(-1)
        assert np.array_equal(got_r[:e - b], col[b:e]) and np.array_equal(got_v[:e - b], valb[b:e]), ("edges of task", op, i)
        assert (got_r[e - b:] == ZERO_ROW).all() and (got_v[e - b:] == 0).all(), ("pad entries of task", op, i)
    assert im["idx"][-1] == ZERO_ROW * 0x01010101 and (im["val"][-1] == 0).all()
    # the longest-first deal: loads as the builder models them, max - min within one warp-task's cost (or warp 0's handicap)
    load = np.zeros(WARPS, dtype=np.int64)
    load[0] = LPT_HANDICAP
    cmax = 0
    for s in range(SEGS):
        for slot, ts in seg_wts[s]:
            c = LPT_A * ng[ts[0]] + LPT_B
            load[slot_warp[slot]] += c
            cmax = max(cmax, c)
    assert load.max() - load.min() <= max(cmax, LPT_HANDICAP), (load, cmax)
    return im


def _dconv_plan(g, n):
    ei, ew = _tensors(g)
    return GraphPlan(_lib.FLAVOR_DCONV, ei, ew, n, flags=_lib.DCONV_ALLOW_DUPLICATES)


@pytest.mark.parametrize("kind,n,edges", GEOMETRIES, ids=GEO_IDS)
def test_graph_image_structure(kind, n, edges):
    g = make_graph(kind, n, edges)
    plan = _dconv_plan(g, n)
    ei, ew = _tensors(g)
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei, ew, n, normalization="sym")
    for p, n_ops in ((plan, 1), (plan, 2), (cheb, 1)):
        nnz = sum(p.nnz(op) for op in range(n_ops))
        fits = image_fits(n, n_ops, nnz)
        assert (p.graph_image(n_ops) is not None) == fits, (n_ops, nnz)
        assert ops.gru_seq_supported(p, n_ops, 2, 32) == fits           # the wgmma kernel takes exactly the plans that have an image
        if fits:
            check_image(p, n_ops)
    if kind == "edges" and edges in (E_DENSE, E_DENSE + 4):
        assert (plan.graph_image(2) is not None) == (edges == E_DENSE)


def test_graph_image_absent():
    src, dst, w = make_graph("random", 208)
    assert _dconv_plan((src, dst, w), 208).graph_image(1) is None       # 8-bit rows and zero row 207: N <= 207 only
    assert _lib.lib().stmp_plan_graph_image(None, 1, None, 0) == 0
    for row_len, has in ((508, True), (509, False)):                    # 7-bit group count: at most 127 groups of four per row
        ring = np.arange(20)
        hub = np.arange(row_len - 1) % 19 + 1                           # duplicate edges into row 0 (BatchedDConv semantics)
        g = (np.concatenate([ring, hub]), np.concatenate([(ring + 1) % 20, np.zeros(row_len - 1, np.int64)]),
             np.ones(19 + row_len, np.float32))
        plan = _dconv_plan(g, 20)
        assert plan.export(0)[0][1].item() == row_len                 # the ring edge 19 -> 0 and the row_len - 1 hub edges
        assert (plan.graph_image(1) is not None) == has and (plan.graph_image(2) is not None) == has
        assert ops.dcrnn_seq_supported(plan, 2, 32, 2)                   # the FFMA kernel still serves it
        if has:
            check_image(plan, 2)
    plan = _dconv_plan(make_graph("ring", 8), 8)
    full = plan.graph_image(2)
    small = torch.full((16,), 0xAB, dtype=torch.uint8)
    size = _lib.lib().stmp_plan_graph_image(plan.handle, 2, ctypes.c_void_p(small.data_ptr()), 16)
    assert size == full.numel() > 16 and (small == 0xAB).all()        # too small a buffer: the size only, nothing copied
    dev = torch.zeros(size, dtype=torch.uint8, device=DEV)              # device destinations work as well
    assert _lib.lib().stmp_plan_graph_image(plan.handle, 2, ctypes.c_void_p(dev.data_ptr()), size) == size
    assert torch.equal(dev.cpu(), full)
    check_image(plan, 2)


# ==== 2. DCRNN forward: wgmma and FFMA kernels against float64 ===========================================================================
def _oracle_dcrnn(sd, X, ei, ew, H0):
    """float64 recurrence from H0 (B, N, 32); with leaf inputs that require grad it is differentiable."""
    B, T, N, F = X.shape
    with _float64():
        ops_ = R.batched_dcrnn_operators(ei, ew.double(), B, N)
        H, outs = H0.reshape(B * N, -1), []
        for t in range(T):
            H = R._dcrnn_step(sd, X[:, t].reshape(B * N, F), ops_, H)
            outs.append(H.reshape(B, N, -1))
    return torch.stack(outs, 1)


def _tiled_dcrnn(m, plan, X, H0):
    H, outs = H0, []
    for t in range(X.size(1)):
        H = m._tiled_step(plan, X[:, t], H)
        outs.append(H)
    return torch.stack(outs, 1)


def _dcrnn_case(n, cin, seed, cout=32, K=2):
    torch.manual_seed(seed)
    m = BatchedDCRNN(cin, cout, K).to(DEV)
    sd64 = {k: v.detach().double() for k, v in m.state_dict().items()}
    return m, sd64


@pytest.mark.parametrize("kind,n,edges", GEOMETRIES, ids=GEO_IDS)
def test_dcrnn_forward_vs_float64(kind, n, edges):
    g = make_graph(kind, n, edges)
    ei, ew = _tensors(g)
    for cin in (1, 2, 3, 4):
        tch = 32 // cin
        Ts = sorted({1, tch - 1, tch, tch + 1, 12} - {0})
        Tmax = max(Ts)
        m, sd64 = _dcrnn_case(n, cin, seed=100 * cin + n)
        plan = m._plan(ei, ew, n)
        gen = torch.Generator(device=DEV).manual_seed(cin)
        X = torch.randn(200, Tmax, n, cin, device=DEV, generator=gen)
        H0 = 0.5 * torch.randn(200, n, 32, device=DEV, generator=gen)
        pick = [0, 199]
        with torch.no_grad():
            ref64 = _oracle_dcrnn(sd64, X[pick].double(), ei, ew, H0[pick].double())
            ref32 = _tiled_dcrnn(m, plan, X[pick], H0[pick])
        tc = ops.gru_seq_supported(plan, 2, cin, 32)
        assert tc == image_fits(n, 2, 2 * len(g[0]))
        with _option("dcrnn_tc", 0, 1):
            ffma_ok = ops.dcrnn_seq_supported(plan, cin, 32, 2)
        for T in Ts:
            for B in (1, 200):
                args = (plan, X[:B, :T], *m._params(), 2)
                res = {}
                if tc:
                    with torch.no_grad(), _counted() as c:
                        res["tc"] = ops.dcrnn_seq_fwd(*args, h0=H0[:B], wimage=m._weight_image())
                    assert c.get("k_dcrnn_seq_tc") == 1 and "k_dcrnn_seq" not in c
                    split = B == 1 and n > 128
                    assert c.get("k_dcrnn_seq_tc[cluster2]", 0) == int(split)
                    if split:                                   # the cluster pair equals one CTA, bit for bit
                        with torch.no_grad(), _option("dcrnn_fwd_split", 0, 1), _counted() as c1:
                            one = ops.dcrnn_seq_fwd(*args, h0=H0[:B], wimage=m._weight_image())
                        assert "k_dcrnn_seq_tc[cluster2]" not in c1
                        assert torch.equal(one, res["tc"]), (cin, T)
                with torch.no_grad(), _option("dcrnn_tc", 0, 1), _counted() as c:
                    try:
                        res["ffma"] = ops.dcrnn_seq_fwd(*args, h0=H0[:B])
                    except _lib.StmpUnsupported:        # the FFMA kernel holds the window's X in shared memory
                        assert not ffma_ok or T > 12, (cin, T)
                if "ffma" in res:
                    assert c.get("k_dcrnn_seq") == 1 and "k_dcrnn_seq_tc" not in c
                for name, out in res.items():
                    sel = [0] if B == 1 else pick
                    _assert_err(out[sel], ref32[:len(sel), :T], ref64[:len(sel), :T], (name, cin, T, B))
                if len(res) == 2:
                    d = float((res["tc"] - res["ffma"]).abs().max())
                    assert d < 2e-5, ("wgmma vs FFMA", cin, T, B, d)
        if not tc:
            assert kind == "edges" and edges > E_DENSE


@pytest.mark.parametrize("n", [32, 33, 64, 65, 128, 129, 224, 225, 256])
def test_dcrnn_ffma_row_mappings_vs_float64(n):
    """k_dcrnn_seq's five row mappings (RT 1/2/4/7 with 8 warps, 4 with 16 warps) at K != 2 and cout 16 / 32."""
    g = make_graph("random", n)
    ei, ew = _tensors(g)
    ran = 0
    for cout in (16, 32):
        for K in (1, 3):
            m, sd64 = _dcrnn_case(n, 2, seed=n + cout + K, cout=cout, K=K)
            plan = m._plan(ei, ew, n)
            gen = torch.Generator(device=DEV).manual_seed(K)
            X = torch.randn(3, 12, n, 2, device=DEV, generator=gen)
            H0 = 0.5 * torch.randn(3, n, cout, device=DEV, generator=gen)
            args = (plan, X, *m._params(), K)
            if not ops.dcrnn_seq_supported(plan, 2, cout, K):
                with pytest.raises(_lib.StmpUnsupported):
                    ops.dcrnn_seq_fwd(*args, h0=H0)
                continue
            with torch.no_grad(), _counted() as c:
                out = ops.dcrnn_seq_fwd(*args, h0=H0)
                ref32 = _tiled_dcrnn(m, plan, X[:2], H0[:2])
            assert c.get("k_dcrnn_seq") == 1 and "k_dcrnn_seq_tc" not in c
            ref64 = _oracle_dcrnn(sd64, X[:2].double(), ei, ew, H0[:2].double())
            _assert_err(out[:2], ref32, ref64, (cout, K))
            ran += 1
    assert ran >= 2 + (n <= 207)


# ==== 3. DCRNN training: the persistent backward, staged and global graph ================================================================
def _train_grads(out, leaves, wgt):
    (out * wgt).mean().backward()
    return [t.grad.detach().clone() for t in leaves]


@pytest.mark.parametrize("kind,n,edges", GEOMETRIES, ids=GEO_IDS)
def test_dcrnn_training_vs_float64(kind, n, edges):
    g = make_graph(kind, n, edges)
    ei, ew = _tensors(g)
    cins = {E_104: (1, 2), E_104 + 1: (1, 2), E_112: (3, 4), E_112 + 1: (3, 4)}.get(edges, (1, 2, 3, 4))
    for cin in cins:
        m, sd64 = _dcrnn_case(n, cin, seed=7 * cin + n)
        plan = m._plan(ei, ew, n)
        if not ops.gru_seq_supported(plan, 2, cin, 32):             # no image: covered by the forward test's FFMA cases
            assert kind == "edges" and edges > E_DENSE
            continue
        assert ops.dcrnn_bwd_supported(plan, cin, 32, 2)
        gen = torch.Generator(device=DEV).manual_seed(cin + n)
        B, T = 3, 5
        X = torch.randn(B, T, n, cin, device=DEV, generator=gen)
        H0 = 0.5 * torch.randn(B, n, 32, device=DEV, generator=gen)
        wgt = torch.randn(B, T, n, 32, device=DEV, generator=gen)
        params = list(m.parameters())
        # float64 oracle with autograd
        leaves64 = [X.double().requires_grad_(True), H0.double().requires_grad_(True)]
        p64 = {k: v.clone().requires_grad_(True) for k, v in sd64.items()}
        out64 = _oracle_dcrnn(p64, leaves64[0], ei, ew, leaves64[1])
        g64 = _train_grads(out64, leaves64 + [p64[k] for k, _ in m.named_parameters()], wgt.double())
        # fp32 op-for-op
        leaves32 = [X.clone().requires_grad_(True), H0.clone().requires_grad_(True)]
        m.zero_grad()
        g32 = _train_grads(_tiled_dcrnn(m, plan, *leaves32), leaves32 + params, wgt)
        # fused, CTA pairs (B < SMs / 2) and one CTA per window
        fused = []
        staged = bwd_staged(n, cin, [plan.nnz(0), plan.nnz(1)])
        for split in (1, 0):
            with _option("dcrnn_fwd_split", split, 1), _option("dcrnn_bwd_split", split, 1), _counted() as c:
                leaves = [X.clone().requires_grad_(True), H0.clone().requires_grad_(True)]
                m.zero_grad()
                out = _DcrnnSeqFn.apply(leaves[0], leaves[1], *m._params(), plan, 2, m._weight_image())
                fused.append([out.detach()] + _train_grads(out, leaves + params, wgt))
            assert c.get("k_dcrnn_seq_tc") == 1 and c.get("k_dcrnn_bwd_seq") == 1, c
            assert c.get("k_dcrnn_bwd_seq[graph-global]", 0) == int(not staged), (cin, plan.nnz(0))
            assert c.get("k_dcrnn_bwd_seq[cluster2]", 0) == int(split == 1 and n >= 16)
            assert c.get("k_dcrnn_seq_tc[cluster2]", 0) == int(split == 1 and n > 128)
        for a, b in zip(*fused):
            assert torch.equal(a, b), ("cluster pair vs one CTA", cin, float((a - b).abs().max()))
        names = ["out", "dX", "dH0"] + [k for k, _ in m.named_parameters()]
        with torch.no_grad():
            ref32_out = _tiled_dcrnn(m, plan, X, H0)
        for name, got, r32, r64 in zip(names, fused[0], [ref32_out] + g32, [out64.detach()] + g64):
            _assert_err(got, r32, r64, (name, cin))
    if edges in (E_104, E_104 + 1, E_112, E_112 + 1):
        # Regression: at the limit itself the CTA pair's backward failed to launch -- its static mbarrier pushed the block past the
        # 227 KB opt-in limit that the staged-copy budget filled exactly -- and the sticky error then failed the next, unrelated launch.
        assert bwd_staged(n, cins[0], [edges, edges]) == (edges in (E_104, E_112))


# ==== 4. GConvGRU on the one-SM kernel: n_ops = 0 and 1, both normalizations ==============================================================
def _oracle_gconv_gru(m, X, ei, ew, H, normalization, grad=False):
    with _float64():
        p = {k: v.detach().double().requires_grad_(grad) for k, v in m.state_dict().items()}
        x = X.detach().double().requires_grad_(grad)
        h = H.detach().double().requires_grad_(grad)
        out = R.gconv_gru_cell(p, x, ei, ew.double(), h, normalization=normalization)
    return out, x, h, p


@pytest.mark.parametrize("kind,n,edges", GEOMETRIES, ids=GEO_IDS)
def test_gconv_gru_forward_vs_float64(kind, n, edges):
    g = make_graph(kind, n, edges)
    ei, ew = _tensors(g)
    for K in (1, 2):
        for norm in ("sym", "rw"):
            cin = 1 + (K + n) % 4
            torch.manual_seed(K + n)
            m = GConvGRU(cin, 32, K, normalization=norm).to(DEV)
            X = torch.randn(n, cin, device=DEV)
            H = 0.5 * torch.randn(n, 32, device=DEV)
            with torch.no_grad(), _counted() as c:
                out = m(X, ei, ew, H)
            assert c.get("k_dcrnn_seq_tc") == 1, (K, norm, c)
            m.fused_training = False
            ref32 = m(X, ei, ew, H)
            ref64 = _oracle_gconv_gru(m, X, ei, ew, H, norm)[0]
            _assert_err(out, ref32, ref64, (K, norm))


@pytest.mark.parametrize("n", [129, 207])
def test_gconv_gru_training_on_hubs_vs_float64(n):
    g = make_graph("hubs", n)
    ei, ew = _tensors(g)
    for cin in (1, 2, 3, 4):
        torch.manual_seed(cin)
        m = GConvGRU(cin, 32, 2).to(DEV)
        X = torch.randn(n, cin, device=DEV)
        H = 0.5 * torch.randn(n, 32, device=DEV)
        wgt = torch.randn(n, 32, device=DEV)
        params = list(m.parameters())
        out64, x64, h64, p64 = _oracle_gconv_gru(m, X, ei, ew, H, "sym", grad=True)
        g64 = _train_grads(out64, [x64, h64] + [p64[k] for k, _ in m.named_parameters()], wgt.double())
        res = []
        for fused in (True, False):
            m.fused_training = fused
            m.zero_grad()
            leaves = [X.clone().requires_grad_(True), H.clone().requires_grad_(True)]
            with _counted() as c:
                out = m(*leaves[:1], ei, ew, leaves[1])
                res.append([out.detach()] + _train_grads(out, leaves + params, wgt))
            if fused:
                plan = m._cheb_plan(ei, ew, n, "sym", None)
                staged = bwd_staged(n, cin, [plan.nnz(0)])
                assert c.get("k_dcrnn_seq_tc") == 1 and c.get("k_gru_bwd_seq") == 1, c
                assert c.get("k_gru_bwd_seq[graph-global]", 0) == int(not staged), (cin, plan.nnz(0))
        names = ["out", "dX", "dH"] + [k for k, _ in m.named_parameters()]
        for name, got, r32, r64 in zip(names, res[0], res[1], [out64.detach()] + g64):
            _assert_err(got, r32, r64, (name, cin))
