"""The row image of the one-CTA wgmma graph-GRU kernel (csrc/row_image.cuh), built on the host by stmp_row_image_build, against a
Python restatement of the builder, plus the properties the kernel relies on: every row once per operator, entries in CSR order,
pad entries on an empty zero row, balanced quads and warps, and refusal of graphs the 8-bit format cannot hold.  Needs no GPU."""
import ctypes

import numpy as np
import pytest

from pytorch_geometric_temporal_b200 import _lib

POS, WARPS, BINS = 256, 16, 32
OFF_PERM, OFF_IPOS, OFF_GSTART, OFF_GCOUNT, OFF_IDX = 16, 16 + 512, 16 + 768, 16 + 768 + 128, 16 + 768 + 256


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def build(n, ops):
    """C builder: ops = [(rowptr, col, val)] * n_ops (numpy).  Returns the image bytes, or None when refused."""
    args = []
    for k in range(2):
        rp, col, val = ops[k] if k < len(ops) else (None, None, None)
        args += [_ptr(rp), _ptr(col), _ptr(val)]
    size = int(_lib.lib().stmp_row_image_build(n, len(ops), *args, None, 0))
    if size == 0:
        return None
    buf = np.zeros(size, np.uint8)
    assert int(_lib.lib().stmp_row_image_build(n, len(ops), *args, _ptr(buf), size)) == size
    return buf.tobytes()


def build_ref(n, ops):
    """Python restatement of plan.cu::build_row_image."""
    n_ops = len(ops)
    ng = np.zeros((2, n), np.int64)
    for op, (rp, _, _) in enumerate(ops):
        ng[op] = (np.diff(rp) + 3) // 4
    cost = ng[0] + ng[1]
    order = sorted(range(n), key=lambda i: -cost[i]) + [-1] * (POS - n)
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


def parse(img):
    hdr = np.frombuffer(img, np.int32, 4)
    n_groups = int(hdr[0])
    perm = np.frombuffer(img, np.int16, POS, OFF_PERM)
    ipos = np.frombuffer(img, np.uint8, POS, OFF_IPOS)
    gstart = np.frombuffer(img, np.uint16, WARPS * 4, OFF_GSTART).reshape(WARPS, 2, 2)
    gcount = np.frombuffer(img, np.uint16, WARPS * 4, OFF_GCOUNT).reshape(WARPS, 2, 2)
    idx = np.frombuffer(img, np.uint32, (n_groups + 1) * 8, OFF_IDX).reshape(-1, 8)
    val = np.frombuffer(img, np.float32, (n_groups + 1) * 32, OFF_IDX + (n_groups + 1) * 32).reshape(-1, 8, 4)
    assert len(img) == OFF_IDX + (n_groups + 1) * 160
    return hdr, perm, ipos, gstart, gcount, idx, val


def random_op(rng, n, max_deg):
    deg = rng.integers(0, max_deg + 1, n)
    deg[rng.integers(0, n)] = 0 if n > 1 else deg[0]
    rp = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    col = np.concatenate([rng.choice(n, d, replace=d > n) for d in deg]).astype(np.int32) if deg.sum() else np.zeros(0, np.int32)
    val = rng.standard_normal(int(deg.sum())).astype(np.float32)
    return rp, col, val


CASES = [(1, 1, 3), (7, 2, 5), (64, 2, 12), (128, 1, 9), (129, 2, 9), (207, 2, 17), (207, 2, 40), (255, 2, 8), (200, 1, 130)]


@pytest.mark.parametrize("n,n_ops,max_deg", CASES)
def test_row_image_matches_restatement_and_invariants(n, n_ops, max_deg):
    rng = np.random.default_rng(n * 131 + n_ops * 7 + max_deg)
    ops = [random_op(rng, n, max_deg) for _ in range(n_ops)]
    img = build(n, ops)
    assert img is not None
    assert img == build_ref(n, ops)
    hdr, perm, ipos, gstart, gcount, idx, val = parse(img)
    n_groups, zero_pos = int(hdr[0]), int(hdr[1])
    assert (int(hdr[2]), int(hdr[3])) == (n, n_ops)
    # every node at exactly one position; ipos inverts perm; the zero row is empty
    nodes = perm[perm >= 0]
    assert sorted(nodes.tolist()) == list(range(n)) and (perm < 0).sum() == POS - n
    assert all(perm[ipos[i]] == i for i in range(n))
    assert perm[zero_pos] == -1
    ng = [(np.diff(rp) + 3) // 4 for rp, _, _ in ops]
    load = np.zeros(WARPS, np.int64)
    for w in range(WARPS):
        for op in range(n_ops):
            rp, col, cval = ops[op]
            for s in range(2):
                g0, G = int(gstart[w, op, s]), int(gcount[w, op, s])
                assert g0 + G <= n_groups
                quad_nodes = [int(perm[16 * w + 8 * s + quad]) for quad in range(8)]
                # a list runs exactly as long as its longest row
                assert G == max([int(ng[op][x]) for x in quad_nodes if x >= 0] + [0])
                load[w] += G
                for quad, node in enumerate(quad_nodes):
                    ent = [((int(idx[g0 + g, quad]) >> (8 * e)) & 0xFF, val[g0 + g, quad, e]) for g in range(G) for e in range(4)]
                    ln = int(rp[node + 1] - rp[node]) if node >= 0 else 0
                    if ln:   # the row's entries, once each, in CSR order, then pads
                        beg = int(rp[node])
                        assert [perm[s_] for s_, _ in ent[:ln]] == col[beg:beg + ln].tolist()
                        assert np.array_equal(np.array([v for _, v in ent[:ln]], np.float32), cval[beg:beg + ln])
                    assert all(s_ == zero_pos and v == 0.0 for s_, v in ent[ln:])
    # the spare group row
    assert (idx[n_groups] == zero_pos * 0x01010101).all() and (val[n_groups] == 0).all()
    # the lists tile the group arrays
    assert int(load.sum()) == n_groups
    # quad balance: the 8 rows of a (warp, slot) are adjacent in the order of their group counts, so the cost ranges of the bins do
    # not overlap and add up to at most the graph's range; warp balance: no warp carries more than one bin's work over another
    cost = ng[0] + (ng[1] if n_ops > 1 else 0)
    spread, bin_costs = 0, []
    for w in range(WARPS):
        for s in range(2):
            q_nodes = [int(x) for x in perm[16 * w + 8 * s:16 * w + 8 * s + 8] if x >= 0]
            if q_nodes:
                spread += int(cost[q_nodes].max() - cost[q_nodes].min())
            bin_costs.append(sum(int(gcount[w, op, s]) for op in range(n_ops)))
    assert spread <= int(cost.max() - cost.min())
    assert load.max() - load.min() <= max(bin_costs)


def test_row_image_single_operator_ignores_the_second_set():
    rng = np.random.default_rng(3)
    op0 = random_op(rng, 50, 6)
    assert build(50, [op0]) == build_ref(50, [op0])


@pytest.mark.parametrize("case", ["n_too_large", "n_zero", "col_out_of_range", "negative_col", "n_ops_3", "rowptr_decreasing"])
def test_row_image_refuses_what_the_format_cannot_hold(case):
    rng = np.random.default_rng(5)
    n = 256 if case == "n_too_large" else 20
    rp, col, val = random_op(rng, n, 4)
    n_ops = 1
    if case == "n_zero":
        n = 0
    elif case == "col_out_of_range":
        col = col.copy(); col[0] = n
    elif case == "negative_col":
        col = col.copy(); col[-1] = -1
    elif case == "n_ops_3":
        n_ops = 3
    elif case == "rowptr_decreasing":
        rp = rp.copy(); rp[3], rp[4] = rp[4] + 1, rp[3]
    args = [_ptr(rp), _ptr(col), _ptr(val), _ptr(rp), _ptr(col), _ptr(val)]
    assert int(_lib.lib().stmp_row_image_build(n, n_ops, *args, None, 0)) == 0
