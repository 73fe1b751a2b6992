"""ASTGCN inference on graphs wider than one spatial-attention row tile: 321 .. 1024 nodes, the PeMS03 / PeMS07 networks.

* the column-tiled spatial-attention pair (stmp_spatial_attention_tiled_fwd: k_spatt_tiles + k_spatt_norm) against float64, with logits
  large enough that a softmax without the max subtraction overflows, exact-zero padding columns, bit-identical repeats, empty batches,
  agreement with the one-tile kernel at 307 nodes, and its argument errors;
* ASTGCN(3 blocks, K=3, 64/64 filters) on the PeMS07 / PeMS03 shapes against the unmodified reference evaluated in float64
  (tests/golden/make_goldens_astgcn_large.py), against the op-for-op path, per-call kernel counts, the routes that stay op-for-op
  (training, edge_index lists, > 1024 nodes) and a captured CUDA graph."""
import ctypes
import gzip
import os

import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN
from pytorch_geometric_temporal_b200.nn.attention import astgcn as astgcn_mod

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ran(c0, name):
    return _lib.path_counters().get(name, 0) - c0.get(name, 0)


def _inputs(n, B, T, seed, vs_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    lhs, rhs = torch.randn(B, n, T, generator=g) * 0.5, torch.randn(B, T, n, generator=g) * 0.5
    bs, Vs = torch.randn(n, n, generator=g) * 0.3, torch.randn(n, n, generator=g) * (1.5 / n ** 0.5) * vs_scale
    return lhs, rhs, bs, Vs


def _want(lhs, rhs, bs, Vs):
    """(float64 softmax_dim1, float32 torch error of the same, max |logit|)"""
    L = Vs.double() @ torch.sigmoid(lhs.double() @ rhs.double() + bs.double())
    S = torch.softmax(L, dim=1)
    S32 = torch.softmax(Vs @ torch.sigmoid(lhs @ rhs + bs), dim=1)
    return S, (S32.double() - S).abs().max().item(), L.abs().max().item()


def _tiled(lhs, rhs, bs, Vs):
    return ops.spatial_attention_tiled(lhs.to(DEV), rhs.to(DEV), bs.t().contiguous().to(DEV), ops.spatial_attention_prepack(Vs.to(DEV)))


KERNEL_CASES = [(321, 1, 12), (321, 3, 7), (358, 1, 1), (358, 3, 12), (358, 32, 12), (383, 1, 7), (383, 3, 1), (512, 1, 12), (512, 3, 7),
                (883, 1, 1), (883, 3, 12), (1024, 1, 7), (1024, 3, 12)]


@pytest.mark.parametrize("n,B,T", KERNEL_CASES)
def test_tiled_spatial_attention_vs_fp64(n, B, T):
    lhs, rhs, bs, Vs = _inputs(n, B, T, 1000 * n + 10 * B + T)
    S, err32, _ = _want(lhs, rhs, bs, Vs)
    P = (n + 63) // 64 * 64
    c0 = _lib.path_counters()
    ST = _tiled(lhs, rhs, bs, Vs)
    assert _ran(c0, "k_spatt_tiles") == 1 and _ran(c0, "k_spatt_norm") == 1
    assert ST.shape == (B, n, P)
    got = ST[:, :, :n].transpose(1, 2).cpu().double()
    err = (got - S).abs().max().item()
    assert err <= 4 * err32 + 2e-6, (n, B, T, err, err32)
    assert torch.all(ST[:, :, n:] == 0)
    assert torch.equal(ST, _tiled(lhs, rhs, bs, Vs))                     # deterministic: no atomics, fixed combine order


@pytest.mark.parametrize("n,B,T", [(358, 3, 12), (883, 2, 12), (1024, 1, 7)])
def test_tiled_spatial_attention_large_logits(n, B, T):
    """logits of magnitude ~50 and more: exp without the max subtraction overflows float32 (e^89 = inf)"""
    lhs, rhs, bs, Vs = _inputs(n, B, T, 7 * n + T, vs_scale=40.0)
    S, err32, lmax = _want(lhs, rhs, bs, Vs)
    assert lmax > 50
    ST = _tiled(lhs, rhs, bs, Vs)
    got = ST[:, :, :n].transpose(1, 2).cpu().double()
    assert torch.isfinite(got).all()
    err = (got - S).abs().max().item()
    assert err <= 4 * err32 + 2e-6, (n, err, err32)
    assert torch.all(ST[:, :, n:] == 0)


def test_tiled_agrees_with_one_tile_kernel_at_307_nodes():
    lhs, rhs, bs, Vs = _inputs(307, 5, 12, 307)
    S, err32, _ = _want(lhs, rhs, bs, Vs)
    c0 = _lib.path_counters()
    one = ops.spatial_attention(lhs.to(DEV), rhs.to(DEV), bs.t().contiguous().to(DEV), ops.spatial_attention_prepack(Vs.to(DEV)))
    assert _ran(c0, "k_gemm_blocks") == 1 and _ran(c0, "k_spatt_tiles") == 0       # <= 320 nodes: the one-tile kernel, as before
    til = _tiled(lhs, rhs, bs, Vs)
    assert (one - til).abs().max().item() <= 4 * err32 + 2e-6
    assert (til[:, :, :307].transpose(1, 2).cpu().double() - S).abs().max().item() <= 4 * err32 + 2e-6
    assert torch.all(til[:, :, 307:] == 0)


def test_spatial_attention_dispatches_above_320_nodes():
    lhs, rhs, bs, Vs = _inputs(400, 2, 12, 3)
    c0 = _lib.path_counters()
    ST = ops.spatial_attention(lhs.to(DEV), rhs.to(DEV), bs.t().contiguous().to(DEV), ops.spatial_attention_prepack(Vs.to(DEV)))
    assert _ran(c0, "k_spatt_tiles") == 1 and _ran(c0, "k_gemm_blocks") == 0
    assert torch.equal(ST, _tiled(lhs, rhs, bs, Vs))


def test_tiled_empty_batch_launches_nothing():
    lhs, rhs, bs, Vs = _inputs(500, 1, 12, 5)
    bsT, packed = bs.t().contiguous().to(DEV), ops.spatial_attention_prepack(Vs.to(DEV))[0]
    n0 = _lib.launch_count()
    ST = ops.spatial_attention_tiled(lhs[:0].to(DEV), rhs[:0].to(DEV), bsT, packed)
    assert ST.shape == (0, 500, 512)
    st = torch.empty(1, 500, 512, device=DEV)
    rc = _lib.lib().stmp_spatial_attention_tiled_fwd(0, 500, 12, _lib.ptr(lhs.to(DEV)), _lib.ptr(rhs.to(DEV)), _lib.ptr(bsT), _lib.ptr(packed),
                                                     _lib.ptr(st), 512, None, 0, _lib.stream_ptr())
    assert rc == _lib.STMP_OK
    assert _lib.launch_count() == n0
    assert _lib.lib().stmp_spatial_attention_tiled_workspace_bytes(0, 500) == 0


def test_tiled_abi_errors():
    n, B, T, P = 700, 2, 12, 704
    lhs, rhs, bs, Vs = _inputs(n, B, T, 9)
    lhs, rhs, bsT = lhs.to(DEV), rhs.to(DEV), bs.t().contiguous().to(DEV)
    packed = ops.spatial_attention_prepack(Vs.to(DEV))[0]
    l = _lib.lib()
    need = l.stmp_spatial_attention_tiled_workspace_bytes(B, n)
    assert need == B * n * 3 * 8                                         # 704 columns: tiles of 256, 256, 192
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    st = torch.empty(B, n, P + 4, device=DEV)
    P_ = _lib.ptr

    def call(B_=B, n_=n, T_=T, lh=lhs, rh=rhs, b=bsT, pk=packed, out=None, ld=P, w=None, wb=need):
        return l.stmp_spatial_attention_tiled_fwd(B_, n_, T_, P_(lh), P_(rh), P_(b), P_(pk), out if out is not None else P_(st), ld,
                                                  P_(ws) if w is None else w, wb, _lib.stream_ptr())

    assert call() == _lib.STMP_OK
    assert call(ld=P + 4) == _lib.STMP_OK
    for kw in (dict(lh=None), dict(rh=None), dict(b=None), dict(pk=None), dict(out=ctypes.c_void_p(0))):
        assert call(**kw) == _lib.STMP_EINVAL, kw
        assert "NULL" in _lib.last_error()
    assert call(w=ctypes.c_void_p(0)) == _lib.STMP_EINVAL
    assert call(wb=need - 8) == _lib.STMP_EINVAL and "workspace" in _lib.last_error()
    assert call(w=ctypes.c_void_p(ws.data_ptr() + 4), wb=need - 4) == _lib.STMP_EINVAL
    assert call(ld=P - 4) == _lib.STMP_ESHAPE
    assert call(ld=P + 2) == _lib.STMP_ESHAPE
    assert call(out=ctypes.c_void_p(st.data_ptr() + 4)) == _lib.STMP_ESHAPE
    assert call(n_=1025) == _lib.STMP_EUNSUPPORTED
    assert call(T_=13) == _lib.STMP_EUNSUPPORTED
    assert call(B_=-1) == _lib.STMP_EINVAL and call(n_=0) == _lib.STMP_EINVAL
    assert l.stmp_spatial_attention_tiled_workspace_bytes(1, 1025) == -1
    with pytest.raises(_lib.StmpUnsupported):
        ops.spatial_attention(torch.zeros(1, 1030, 12, device=DEV), torch.zeros(1, 12, 1030, device=DEV), torch.zeros(1030, 1030, device=DEV),
                              ops.spatial_attention_prepack(torch.zeros(1030, 1030, device=DEV)))
    torch.cuda.synchronize()


# ---- the module ------------------------------------------------------------------------------------------------------------------
def _golden(golden_dir):
    with gzip.open(os.path.join(golden_dir, "astgcn_large.pt.gz"), "rb") as f:
        return torch.load(f, weights_only=False)


def _model(g, c):
    """the reference module's parameters: the same init stream under the same seed (checked against the stored checksum)"""
    n = c["X"].size(1)
    torch.manual_seed(c["seed"])
    m = ASTGCN(**g["ctor"], num_of_vertices=n, normalization=c["normalization"])
    chk = float(sum(v.double().abs().sum() for v in m.state_dict().values()))
    assert abs(chk - c["state_checksum"]) <= 1e-6 * c["state_checksum"], "parameter init stream differs from the reference module's"
    return m.to(DEV)


def _close(got, want, rtol=1e-4, atol=1e-5):
    got = got.detach().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


@pytest.mark.parametrize("case", ["pems07_sym", "pems07_none", "pems03_sym"])
def test_astgcn_large_vs_reference_golden(golden_dir, case, monkeypatch):
    g = _golden(golden_dir)
    c = g["cases"][case]
    m = _model(g, c)
    ei, X = c["edge_index"].to(DEV), c["X"].to(DEV)
    c0 = _lib.path_counters()
    with torch.no_grad():
        out = m(X, ei)
    assert _ran(c0, "k_astgcn_factors") == 3
    assert _ran(c0, "k_spatt_tiles") == 3 and _ran(c0, "k_spatt_norm") == 3
    assert _ran(c0, "k_gemm_blocks") == 3 * 2 + 1       # per block: Chebyshev contraction, time conv; + final conv
    assert _ran(c0, "k_spmm") == 6                      # per block: attention-weighted hop + plain hop
    _close(out, c["out"])
    # the op-for-op path (native path off) computes the same
    monkeypatch.setattr(astgcn_mod.ASTGCNBlock, "_native_ok", lambda self, N, Fi, T: False)
    c0 = _lib.path_counters()
    with torch.no_grad():
        ref = m(X, ei)
    assert _ran(c0, "k_spatt_tiles") == 0 and _ran(c0, "k_gemm_blocks") == 0
    _close(ref, c["out"], rtol=2e-4, atol=2e-5)
    _close(out, ref.cpu(), rtol=2e-4, atol=2e-5)


def test_astgcn_large_unchanged_routes(golden_dir):
    g = _golden(golden_dir)
    c = g["cases"]["pems07_sym"]
    m = _model(g, c)
    ei, X = c["edge_index"].to(DEV), c["X"][:2].to(DEV)
    with torch.no_grad():
        native = m(X, ei)
    # training: autograd through the op-for-op path, no tiled kernels
    c0 = _lib.path_counters()
    out = m(X, ei)
    assert out.requires_grad
    assert _ran(c0, "k_spatt_tiles") == 0 and _ran(c0, "k_spatt_norm") == 0 and _ran(c0, "k_gemm_blocks") == 0
    _close(out, native.cpu(), rtol=2e-4, atol=2e-5)
    out.square().mean().backward()
    assert m._blocklist[0]._spatial_attention._Vs.grad is not None
    # a per-timestep edge_index list
    c0 = _lib.path_counters()
    with torch.no_grad():
        out_l = m(X, [ei] * X.size(-1))
    assert _ran(c0, "k_spatt_tiles") == 0 and _ran(c0, "k_gemm_blocks") == 0
    _close(out_l, native.cpu(), rtol=2e-4, atol=2e-5)
    # more than 1024 nodes
    n = 1100
    e = torch.from_numpy(synthetic.random_digraph(n, 2 * n, False, 1)[0]).to(DEV)
    e = torch.cat([e, e.flip(0)], dim=1)
    torch.manual_seed(4)
    big = ASTGCN(**g["ctor"], num_of_vertices=n, normalization="sym").to(DEV)
    c0 = _lib.path_counters()
    with torch.no_grad():
        y = big(torch.randn(1, n, 1, 12, device=DEV), e)
    assert y.shape == (1, n, 12) and torch.isfinite(y).all()
    assert _ran(c0, "k_spatt_tiles") == 0 and _ran(c0, "k_gemm_blocks") == 0 and _ran(c0, "k_astgcn_factors") == 0


def _capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    return graph, out


def test_astgcn_large_cuda_graph_replay(golden_dir):
    """A no_grad forward at 883 nodes captures and replays.  The tiled pair is bit-identical between eager and replay; the whole model
    agrees to rounding only, because the factors kernel (k_astgcn_factors) reduces through shared-memory atomics and its last bits vary
    from run to run (two eager calls differ by ~5e-7) -- at 307 nodes as well."""
    g = _golden(golden_dir)
    c = g["cases"]["pems07_sym"]
    m = _model(g, c)
    ei = c["edge_index"].to(DEV)
    X = c["X"].to(DEV).clone()
    with torch.no_grad():
        blk = m._blocklist[0]
        ta, sa = blk._temporal_attention, blk._spatial_attention
        lhs, rhs = ops.astgcn_factors(X.permute(0, 1, 3, 2).contiguous(), ta._U1, ta._U2, ta._U3, ta._be, ta._Ve, sa._W1, sa._W2, sa._W3)
        pk = blk._native_packs()
        st_eager = ops.spatial_attention(lhs, rhs, pk["bsT"], pk["vsT"])
        g_st, st_static = _capture(lambda: ops.spatial_attention(lhs, rhs, pk["bsT"], pk["vsT"]))
        g_st.replay()
        torch.cuda.synchronize()
        assert torch.equal(st_static, st_eager)

        graph, static_out = _capture(lambda: m(X, ei))
        X.copy_(torch.randn(X.shape, generator=torch.Generator().manual_seed(5)).to(DEV))
        graph.replay()
        eager = m(X, ei)
        torch.cuda.synchronize()
    assert not torch.allclose(eager.cpu(), c["out"], rtol=1e-2, atol=1e-2)   # the replay read the new X
    _close(static_out, eager.cpu(), rtol=1e-5, atol=2e-6)
