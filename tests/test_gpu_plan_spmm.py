"""GPU parity through the C ABI: cached graph operators (K2) and the gather/scatter product (K1/K3).
Index work is BIT-EXACT; SpMM values are bit-exact too because the kernel sums each destination in the
reference's scatter order with separate multiply/add."""
import numpy as np
import pytest
import torch

from oracle import pyg, recurrent as R, attention as A
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.plan import GraphPlan

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _coo_to_ref_csr(n, dst, src, val):
    """Stable sort of a reference-order COO list by destination."""
    order = torch.sort(dst, stable=True).indices
    rowptr = torch.zeros(n + 1, dtype=torch.int64)
    rowptr[1:] = torch.bincount(dst, minlength=n).cumsum(0)
    return rowptr.int(), src[order].int(), val[order], order.int()


def _check_plan(plan, op, n, dst, src, val, exact=True):
    rp, col, v, eid = [t.cpu() for t in plan.export(op)]
    wrp, wcol, wv, weid = _coo_to_ref_csr(n, dst, src, val)
    assert torch.equal(rp, wrp) and torch.equal(col, wcol) and torch.equal(eid, weid)
    if exact:
        assert torch.equal(v, wv), (v - wv).abs().max()
    else:
        assert torch.allclose(v, wv, rtol=1e-6, atol=0)
    # transposed operator: CSR by source
    rp, col, v2, eid = [t.cpu() for t in plan.export(op, transposed=True)]
    wrp, wcol, wv, weid = _coo_to_ref_csr(n, src, dst, val)
    assert torch.equal(rp, wrp) and torch.equal(col, wcol) and torch.equal(eid, weid)


def _graphs():
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    yield "metr_la", 207, torch.from_numpy(ei), torch.from_numpy(ew)
    g = torch.Generator().manual_seed(5)
    n = 50
    ei = torch.randint(0, n, (2, 300), generator=g)  # duplicates + self loops + isolated nodes possible
    yield "random_dups", n, ei, torch.rand(300, generator=g) + 0.1
    ei, ew = synthetic.large_graph(3000, 20000, 1)
    yield "large", 3000, torch.from_numpy(ei), torch.from_numpy(ew)


@pytest.mark.parametrize("name,n,ei,ew", list(_graphs()), ids=lambda v: v if isinstance(v, str) else None)
def test_dconv_plan_bit_exact(name, n, ei, ew):
    dup = name == "random_dups"
    flags = _lib.DCONV_ALLOW_DUPLICATES if dup else 0
    plan = GraphPlan(_lib.FLAVOR_DCONV, ei.to(DEV), ew.to(DEV), n, flags=flags)
    assert plan.n_ops == 2
    eo, no, ei_in, ni = R.dconv_operators(ei, ew, batched=True, num_nodes=n)
    _check_plan(plan, 0, n, eo[1], eo[0], no)
    if not dup:  # argsort tie order of duplicate (col,row) keys is unspecified in the reference
        _check_plan(plan, 1, n, ei_in[1], ei_in[0], ni)
    # edge_weight=None => ones
    plan1 = GraphPlan(_lib.FLAVOR_DCONV, ei.to(DEV), None, n, flags=flags)
    eo, no, _, _ = R.dconv_operators(ei, torch.ones(ei.size(1)), batched=True, num_nodes=n)
    _check_plan(plan1, 0, n, eo[1], eo[0], no)


def test_dconv_plan_matches_dense_adjacency_semantics():
    """DConv proper (dense adjacency + nonzero, dcrnn.py:59-77) on a duplicate-free graph gives the same
    operators as the scatter formulation up to degree rounding."""
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
    plan = GraphPlan(_lib.FLAVOR_DCONV, ei.to(DEV), ew.to(DEV), 207)
    eo, no, ei_in, ni = R.dconv_operators(ei, ew, batched=False, num_nodes=207)
    _check_plan(plan, 0, 207, eo[1], eo[0], no, exact=False)
    _check_plan(plan, 1, 207, ei_in[1], ei_in[0], ni, exact=False)


def test_dconv_duplicates_rejected_like_reference():
    ei = torch.tensor([[0, 0, 1, 2], [1, 1, 2, 0]], device=DEV)
    with pytest.raises(RuntimeError, match="duplicate"):
        GraphPlan(_lib.FLAVOR_DCONV, ei, None, 3)
    with pytest.raises(RuntimeError, match="outside"):
        GraphPlan(_lib.FLAVOR_DCONV, torch.tensor([[0, 5], [1, 2]], device=DEV), None, 3)


@pytest.mark.parametrize("norm", ["sym", "rw", None])
@pytest.mark.parametrize("lam", [None, 2.7])
@pytest.mark.parametrize("name,n,ei,ew", list(_graphs()), ids=lambda v: v if isinstance(v, str) else None)
def test_cheb_plan_bit_exact(name, n, ei, ew, norm, lam):
    plan = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), n, normalization=norm, lambda_max=lam)
    ei2, w2 = pyg.cheb_norm(ei, n, ew, norm, None if lam is None else torch.tensor(lam), torch.float32)
    _check_plan(plan, 0, n, ei2[1], ei2[0], w2)
    plan = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), None, n, normalization=norm, lambda_max=lam)
    ei2, w2 = pyg.cheb_norm(ei, n, None, norm, None if lam is None else torch.tensor(lam), torch.float32)
    _check_plan(plan, 0, n, ei2[1], ei2[0], w2)


@pytest.mark.parametrize("improved", [False, True])
@pytest.mark.parametrize("asl", [True, False])
@pytest.mark.parametrize("name,n,ei,ew", list(_graphs()), ids=lambda v: v if isinstance(v, str) else None)
def test_gcn_plan_bit_exact(name, n, ei, ew, improved, asl):
    if name == "random_dups" and asl:
        # several self loops on one node: torch's indexed assignment keeps an unspecified one; make loops unique
        keep = torch.ones(ei.size(1), dtype=torch.bool)
        seen = set()
        for i, (r, c) in enumerate(ei.t().tolist()):
            if r == c:
                if r in seen:
                    keep[i] = False
                seen.add(r)
        ei, ew = ei[:, keep], ew[keep]
    flags = (_lib.GCN_IMPROVED if improved else 0) | (0 if asl else _lib.GCN_NO_SELF_LOOPS)
    plan = GraphPlan(_lib.FLAVOR_GCN, ei.to(DEV), ew.to(DEV), n, flags=flags)
    ei2, w2 = pyg.gcn_norm(ei, ew, n, improved, asl)
    _check_plan(plan, 0, n, ei2[1], ei2[0], w2)


@pytest.mark.parametrize("norm", ["sym", "rw", None])
def test_cheb_att_plan_bit_exact(norm):
    ei = torch.from_numpy(synthetic.pems04_like(0))
    lam = torch.tensor(2.0 if norm == "sym" else 3.1)
    plan = GraphPlan(_lib.FLAVOR_CHEB_ATT, ei.to(DEV), None, 307, normalization=norm, lambda_max=float(lam))
    ei2, w2 = A.cheb_att_norm(ei, 307, None, norm, lam)
    assert ei2.size(1) == 680 + 2 * 307  # astgcn.py:110 comment: E + N + N
    _check_plan(plan, 0, 307, ei2[0], ei2[1], w2)  # propagated on the transposed index (:167)


@pytest.mark.parametrize("F", [1, 2, 3, 34, 32, 64, 128, 200])
@pytest.mark.parametrize("batch", [None, 3])
def test_spmm_bit_exact_vs_scatter_add(F, batch):
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
    plan = GraphPlan(_lib.FLAVOR_DCONV, ei.to(DEV), ew.to(DEV), 207)
    ops_ = R.dconv_operators(ei, ew, batched=True, num_nodes=207)
    g = torch.Generator().manual_seed(F)
    x = torch.randn((207, F) if batch is None else (batch, 207, F), generator=g)
    for op, (e, w) in enumerate(((ops_[0], ops_[1]), (ops_[2], ops_[3]))):
        want = pyg.propagate(e, x, w)
        got = ops.spmm_raw(plan, op, x.to(DEV)).cpu()
        assert torch.equal(got, want), (got - want).abs().max()
        # fused Chebyshev axpby: 2*prop(x) - z  (dcrnn.py:96)
        z = torch.randn(x.shape, generator=g)
        want2 = 2.0 * pyg.propagate(e, x, w) - z
        got2 = ops.spmm_raw(plan, op, x.to(DEV), alpha=2.0, z=z.to(DEV), beta=-1.0).cpu()
        assert torch.equal(got2, want2)
        # transposed product == propagate on the reversed edge list (up to summation order)
        wt = pyg.propagate(e[[1, 0]], x, w)
        gt = ops.spmm_raw(plan, op, x.to(DEV), transposed=True).cpu()
        assert torch.allclose(gt, wt, rtol=1e-5, atol=1e-6)


def test_spmm_large_graph_and_strided_views():
    ei, ew = synthetic.large_graph(10000, 100000, 0)
    ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
    plan = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 10000, normalization="sym")
    ei2, w2 = pyg.cheb_norm(ei, 10000, ew, "sym", None, torch.float32)
    x = torch.randn(2, 10000, 64)
    want = pyg.propagate(ei2, x, w2)
    assert torch.equal(ops.spmm_raw(plan, 0, x.to(DEV)).cpu(), want)


def test_spmm_attention_weighted():
    ei = torch.from_numpy(synthetic.pems04_like(0))
    plan = GraphPlan(_lib.FLAVOR_CHEB_ATT, ei.to(DEV), None, 307, normalization="sym")
    ei2, norm = A.cheb_att_norm(ei, 307, None, "sym", torch.tensor(2.0))
    B, F = 4, 5
    x, S = torch.randn(B, 307, F), torch.rand(B, 307, 307)
    att = norm * S[:, ei2[0], ei2[1]]
    want = pyg.propagate(ei2[[1, 0]], x, att)
    got = ops.spmm_raw(plan, 0, x.to(DEV), att=S.to(DEV)).cpu()
    assert torch.equal(got, want), (got - want).abs().max()


def test_spmm_autograd_matches_oracle_autograd():
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
    plan = GraphPlan(_lib.FLAVOR_DCONV, ei.to(DEV), ew.to(DEV), 207)
    o = R.dconv_operators(ei, ew, batched=True, num_nodes=207)
    x = torch.randn(2, 207, 8, requires_grad=True)
    z = torch.randn(2, 207, 8, requires_grad=True)
    wgt = torch.randn(2, 207, 8)
    (2.0 * pyg.propagate(o[2], x, o[3]) - z).mul(wgt).sum().backward()
    xg = x.detach().to(DEV).requires_grad_(True)
    zg = z.detach().to(DEV).requires_grad_(True)
    ops.spmm(plan, 1, xg, alpha=2.0, z=zg, beta=-1.0).mul(wgt.to(DEV)).sum().backward()
    assert torch.allclose(xg.grad.cpu(), x.grad, rtol=1e-5, atol=1e-6)
    assert torch.allclose(zg.grad.cpu(), z.grad, rtol=1e-6, atol=1e-7)


def test_window_gather_bit_exact():
    from oracle import signal as OS
    series = torch.randn(80, 207, 2)
    starts = torch.tensor([0, 5, 17, 56, 3])
    x, y = ops.window_gather(series.to(DEV), starts.to(DEV), 12)
    for b, s in enumerate(starts.tolist()):
        wx, wy = OS.index_window(series, [s], 0, 12)
        assert torch.equal(x[b].cpu(), wx) and torch.equal(y[b].cpu(), wy)
    series3 = torch.randn(40, 7, 3)  # row not a multiple of 4 floats -> scalar path
    x, y = ops.window_gather(series3.to(DEV), starts[:3].to(DEV), 4)
    assert torch.equal(x[2].cpu(), series3[17:21]) and torch.equal(y[1].cpu(), series3[9:13])


def test_device_prefetcher_slow_consumer_never_sees_a_torn_batch():
    """The H2D copy of batch i+2 reuses the staging buffer of batch i: it must wait for the consumer kernels of batch i
    (enqueued on the compute stream) -- checked with a consumer that is much slower than the copies and a host that runs
    far ahead of the GPU."""
    from pytorch_geometric_temporal_b200.signal import DevicePrefetcher
    n, shape = 12, (1 << 20,)
    host = [torch.full(shape, float(i)).pin_memory() for i in range(n)]
    spin = torch.randn(2048, 2048, device=DEV)
    sums = []
    for i, xb in enumerate(DevicePrefetcher(iter(host), DEV)):
        for _ in range(6):                      # slow consumer: several GEMMs enqueued before the batch is read
            spin = torch.tanh(spin @ spin) * 0.5
        sums.append((xb.sum(), xb.min(), xb.max()))      # reads the staging buffer late on the compute stream
    torch.cuda.synchronize()
    for i, (s, lo, hi) in enumerate(sums):
        assert float(lo) == float(hi) == float(i), (i, float(lo), float(hi))
        assert float(s) == float(i) * shape[0]


def test_index_batch_loader_host_batches_and_forward_indexed_match_materialised_windows():
    """e2e shape of bench.py: window starts from the host -> DevicePrefetcher -> forward_indexed == forward on gathered windows."""
    from pytorch_geometric_temporal_b200.dataset import synthetic
    from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN
    from pytorch_geometric_temporal_b200.signal import DevicePrefetcher, IndexBatchLoader, index_splits
    ei, ew, series = synthetic.metr_la_like(0, 128)
    ei_t, ew_t, sd = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV), torch.from_numpy(series).to(DEV)
    tr, _, _ = index_splits(128, 12)
    loader = IndexBatchLoader(sd, tr, 12, 16, shuffle=True, seed=3, drop_last=True, materialize=False)
    mat = IndexBatchLoader(sd, tr, 12, 16, shuffle=True, seed=3, drop_last=True, materialize=True)
    m = BatchedDCRNN(2, 32, 2).to(DEV)
    with torch.no_grad():
        for st, (x, _) in zip(DevicePrefetcher(loader.host_batches(), DEV), mat):
            assert st.dtype == torch.int64 and st.numel() == 16
            assert torch.equal(m.forward_indexed(sd, st, 12, ei_t, ew_t), m(x, ei_t, ew_t))


# ---- K4: wgmma split-fp16 GEMM (stmp_gemm_f32) and its fused LSTM epilogue ------------------------------------------
@pytest.mark.parametrize("M,K,N", [(1, 4, 32), (127, 36, 64), (128, 64, 96), (1000, 384, 256), (20000, 132, 128)])
def test_gemm_tc_matches_fp64(M, K, N):
    g = torch.Generator().manual_seed(M + K + N)
    A = torch.randn(M, K, generator=g) * 2
    W = (torch.rand(K, N, generator=g) - 0.5) * 0.4
    bias = torch.randn(N, generator=g)
    want64 = A.double() @ W.double() + bias.double()
    packed = ops.gemm_prepack(W.to(DEV))
    got = ops.gemm(A.to(DEV), packed, K, N, bias.to(DEV)).cpu()
    ref32 = A @ W + bias                      # the CPU fp32 result's own error vs fp64 is the yardstick
    err, err32 = (got.double() - want64).abs().max().item(), (ref32.double() - want64).abs().max().item()
    assert err < 4 * err32 + 1e-6, (err, err32)         # fp32-class accuracy: within a small factor of fp32's own error
    assert torch.allclose(got, ref32, rtol=1e-4, atol=1e-4)
    got_nb = ops.gemm(A.to(DEV), packed, K, N).cpu()
    assert torch.allclose(got_nb, A @ W, rtol=1e-4, atol=1e-4)


def test_gemm_tc_rejects_unsupported_shapes():
    W = torch.randn(10, 40, device=DEV)            # N % 32 != 0
    packed = ops.gemm_prepack(W)
    with pytest.raises(_lib.StmpUnsupported):
        ops.gemm(torch.randn(5, 10, device=DEV), packed, 10, 40)
