"""The row image the plan gives the one-CTA wgmma graph-GRU kernel (csrc/row_image.cuh): nodes sorted by operator 0's group count,
then operator 1's, before they are cut into bins of 8 (stmp_row_image_build_by_operator).  Checked against a Python restatement, for
the same structural properties as the by-total image of test_row_image_cpu.py, and for the balance it buys on the benchmark's graph.
Needs no GPU."""
import numpy as np
import pytest

from pytorch_geometric_temporal_b200 import _lib
from pytorch_geometric_temporal_b200.dataset import synthetic
from test_row_image_cpu import BINS, CASES, POS, WARPS, _ptr, build_ref, parse, random_op


def build(n, ops, entry="stmp_row_image_build_by_operator"):
    args = []
    for k in range(2):
        rp, col, val = ops[k] if k < len(ops) else (None, None, None)
        args += [_ptr(rp), _ptr(col), _ptr(val)]
    fn = getattr(_lib.lib(), entry)
    size = int(fn(n, len(ops), *args, None, 0))
    if size == 0:
        return None
    buf = np.zeros(size, np.uint8)
    assert int(fn(n, len(ops), *args, _ptr(buf), size)) == size
    return buf.tobytes()


def build_ref_by_operator(n, ops):
    """Python restatement of plan.cu::build_row_image with ROW_ORDER_BY_OPERATOR: as test_row_image_cpu.build_ref but for the order."""
    n_ops = len(ops)
    ng = np.zeros((2, n), np.int64)
    for op, (rp, _, _) in enumerate(ops):
        ng[op] = (np.diff(rp) + 3) // 4
    order = sorted(range(n), key=lambda i: (-ng[0][i], -ng[1][i])) + [-1] * (POS - n)
    bin_g = np.zeros((BINS, 2), np.int64)
    for k in range(BINS):
        for node in order[8 * k:8 * k + 8]:
            if node >= 0:
                bin_g[k] = np.maximum(bin_g[k], ng[:, node])
    bin_cost = bin_g.sum(1)
    load, used, bin_at = [0] * WARPS, [0] * WARPS, [[None, None] for _ in range(WARPS)]
    for k in sorted(range(BINS), key=lambda k: -bin_cost[k]):
        w = min((w for w in range(WARPS) if used[w] < 2), key=lambda w: load[w])
        bin_at[w][used[w]] = k
        used[w] += 1
        load[w] += int(bin_cost[k])
    perm = np.full(POS, -1, np.int16)
    ipos = np.zeros(POS, np.uint8)
    for w in range(WARPS):
        for s in range(2):
            for quad in range(8):
                node = order[8 * bin_at[w][s] + quad]
                perm[16 * w + 8 * s + quad] = node
                if node >= 0:
                    ipos[node] = 16 * w + 8 * s + quad
    zero_pos = int(np.nonzero(perm < 0)[0][0])
    gstart = np.zeros((WARPS, 2, 2), np.uint16)
    gcount = np.zeros((WARPS, 2, 2), np.uint16)
    idx, vals = [], []
    run = 0
    for w in range(WARPS):
        for op in range(n_ops):
            rp, col, val = ops[op]
            for s in range(2):
                G = int(bin_g[bin_at[w][s], op])
                gstart[w, op, s], gcount[w, op, s] = run, G
                for g in range(G):
                    row_i, row_v = [], []
                    for quad in range(8):
                        node = int(perm[16 * w + 8 * s + quad])
                        beg, ln = (int(rp[node]), int(rp[node + 1] - rp[node])) if node >= 0 else (0, 0)
                        u, vv = 0, []
                        for e in range(4):
                            k = 4 * g + e
                            u |= (int(ipos[col[beg + k]]) if k < ln else zero_pos) << (8 * e)
                            vv.append(val[beg + k] if k < ln else 0.0)
                        row_i.append(u)
                        row_v.append(vv)
                    idx.append(row_i)
                    vals.append(row_v)
                run += G
    idx.append([zero_pos * 0x01010101] * 8)
    vals.append([[0.0] * 4] * 8)
    head = np.array([run, zero_pos, n, n_ops], np.int32).tobytes()
    return (head + perm.tobytes() + ipos.tobytes() + gstart.tobytes() + gcount.tobytes()
            + np.array(idx, np.uint32).tobytes() + np.array(vals, np.float32).tobytes())



def check_rows(n, ops, img):
    """Every node at one position, every row of every operator once in CSR order, then pads on the empty zero row."""
    hdr, perm, ipos, gstart, gcount, idx, val = parse(img)
    n_groups, zero_pos = int(hdr[0]), int(hdr[1])
    assert sorted(perm[perm >= 0].tolist()) == list(range(n)) and all(perm[ipos[i]] == i for i in range(n))
    assert perm[zero_pos] == -1
    load = np.zeros(WARPS, np.int64)
    for w in range(WARPS):
        for op, (rp, col, cval) in enumerate(ops):
            for s in range(2):
                g0, G = int(gstart[w, op, s]), int(gcount[w, op, s])
                load[w] += G
                for quad in range(8):
                    node = int(perm[16 * w + 8 * s + quad])
                    ln = int(rp[node + 1] - rp[node]) if node >= 0 else 0
                    assert ln <= 4 * G
                    ent = [((int(idx[g0 + g, quad]) >> (8 * e)) & 0xFF, val[g0 + g, quad, e]) for g in range(G) for e in range(4)]
                    beg = int(rp[node]) if node >= 0 else 0
                    assert [perm[x] for x, _ in ent[:ln]] == col[beg:beg + ln].tolist()
                    assert np.array_equal(np.array([v for _, v in ent[:ln]], np.float32), cval[beg:beg + ln])
                    assert all(x == zero_pos and v == 0.0 for x, v in ent[ln:])
    assert int(load.sum()) == n_groups
    return load


@pytest.mark.parametrize("n,n_ops,max_deg", CASES)
def test_by_operator_image_matches_restatement_and_rows(n, n_ops, max_deg):
    rng = np.random.default_rng(n * 131 + n_ops * 7 + max_deg)
    ops = [random_op(rng, n, max_deg) for _ in range(n_ops)]
    img = build(n, ops)
    assert img is not None and img == build_ref_by_operator(n, ops)
    check_rows(n, ops, img)
    if n_ops == 1:   # one operator: both orders are the order of its group counts
        assert img == build(n, ops, "stmp_row_image_build")


def _bench_ops(seed):
    """The two DConv operators of the benchmark's graph (row = destination, CSR by source order); only their row lengths matter here."""
    ei, ew, _ = synthetic.metr_la_like(seed, 16)
    n = 207
    ops = []
    for src, dst in ((0, 1), (1, 0)):
        s, d = ei[src], ei[dst]
        o = np.lexsort((np.arange(len(d)), d))
        rp = np.concatenate([[0], np.cumsum(np.bincount(d, minlength=n))]).astype(np.int32)
        ops.append((rp, s[o].astype(np.int32), ew[o].astype(np.float32)))
    return n, ops


@pytest.mark.parametrize("seed", [0, 4])
def test_by_operator_image_balances_the_bench_graph(seed):
    """On the benchmark's graph the slowest warp walks 10 group rows per gather round (both operators) against 12 with the by-total
    order, and all warps together 135-137 against 157-158: fewer pad entries, the same real ones."""
    n, ops = _bench_ops(seed)
    new = check_rows(n, ops, build(n, ops))
    old = check_rows(n, ops, build(n, ops, "stmp_row_image_build"))
    assert new.max() == 10 and old.max() == 12, (new.max(), old.max())
    assert new.sum() < old.sum() - 15, (new.sum(), old.sum())


def test_by_operator_image_refuses_what_the_format_cannot_hold():
    rng = np.random.default_rng(5)
    rp, col, val = random_op(rng, 20, 4)
    bad = col.copy()
    bad[0] = 20
    for n, c in ((256, col), (0, col), (20, bad)):
        args = [_ptr(rp), _ptr(c), _ptr(val)] * 2
        assert int(_lib.lib().stmp_row_image_build_by_operator(n, 1, *args, None, 0)) == 0
