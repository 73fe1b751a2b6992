"""GMAN on the H100: every golden case on both routes (the fused attention kernels and op for op), in train and eval mode, against the
reference's float64 values; the attention kernels alone against float64 across their envelope (node counts, head widths 1..16, head
counts, sequence lengths, the mask, logits past 80 in magnitude, every dQ / dK / dV subset); a training forward bit-equal to the no_grad
call, repeatable backwards and loss-scale equivariance; exact launch counts; the spatial attention's peak memory at the PEMS-BAY shape;
CUDA-graph replay of a training step; the routes outside the envelope and the ABI's errors.

The criterion, per tensor (DESIGN §5): the fused route's largest error against float64 is at most 4 times the float32 op-for-op route's
plus 2^-20 of the tensor's largest float64 magnitude.  The goldens other than the costs are held to the same criterion through their
fingerprints (four fixed projections and the norm), with the norm as the scale.  Every Conv2D bias of GMAN sits in front of a BatchNorm,
so its gradient is zero in exact arithmetic: both routes must give zero to 2^-16 of the case's largest gradient."""
import copy
import ctypes
import os

import pytest
import torch

from gman_seq import CASES, fingerprint, load, model_for, run
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.attention import GMAN
from pytorch_geometric_temporal_b200.nn.attention import gman as G
from test_gpu_rows_envelope import _counted

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ALL = ("k_gman_attn_long_fwd", "k_gman_attn_long_bwd_q", "k_gman_attn_long_bwd_kv", "k_gman_attn_short_fwd", "k_gman_attn_short_bwd")


@pytest.fixture(autouse=True)
def _fp32():
    """cuBLAS in full fp32 on the op-for-op route."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _ran(c):
    return {k: v for k, v in c.items() if k in ALL}


def _criterion(fused, op, want, what, scale=None):
    fused, op, want = (t.detach().double().cpu() for t in (fused, op, want))
    assert fused.shape == want.shape == op.shape, (what, fused.shape, want.shape)
    if want.numel() == 0:
        return
    scale = float(want.abs().max()) if scale is None else scale
    ef, eo = float((fused - want).abs().max()), float((op - want).abs().max())
    assert ef <= 4 * eo + 2.0 ** -20 * scale, (what, ef, eo, scale)


def _run_route(c, fused):
    m = model_for(c, GMAN, DEV, torch.float32)
    m.fused_training = fused
    with _counted() as cnt:
        got = run(m, c, DEV, torch.float32)
    torch.cuda.synchronize()
    return got, _ran(cnt)


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_both_routes(name):
    c = load(GOLDEN)["cases"][name]
    gf, ran_f = _run_route(CASES[name], True)
    go, ran_o = _run_route(CASES[name], False)
    L = CASES[name]["L"]
    # op for op in training; the eval call (no_grad) runs fused on both routes
    assert set(ran_o) <= {"k_gman_attn_long_fwd", "k_gman_attn_short_fwd"}, ran_o
    assert ran_f.get("k_gman_attn_long_bwd_kv") == 2 * L * CASES[name]["steps"], ran_f
    assert set(gf) == set(c["fingerprints"]), (sorted(gf), sorted(c["fingerprints"]))
    gscale = max(float(fp[-1]) for k, fp in c["fingerprints"].items() if k.startswith("grad."))
    for k, fp in c["fingerprints"].items():
        if k.startswith("buf.") and k.endswith("num_batches_tracked"):
            assert int(gf[k]) == int(go[k]) == int(c["values"][k]), k
            continue
        if k.startswith("grad.") and k.endswith("_conv2d.bias"):
            assert float(gf[k].abs().max()) <= 2.0 ** -16 * gscale and float(go[k].abs().max()) <= 2.0 ** -16 * gscale, k
            continue
        if k in c["values"]:
            _criterion(gf[k], go[k], c["values"][k].double(), k)
        else:
            _criterion(fingerprint(gf[k]), fingerprint(go[k]), fp, k, scale=float(fp[-1]))


# ---- the kernels alone against float64 -------------------------------------------------------------------------------------------------
def _qkv(B, Tq, Tk, N, K, d, seed, amp=1.0):
    """Signed Q, K, V (not ReLU'd: the kernels must not rely on Q, K, V >= 0), float32 values."""
    g = torch.Generator().manual_seed(seed)
    f = lambda T: torch.randn(B, T, N, K * d, generator=g) * amp
    return f(Tq), f(Tk), torch.randn(B, Tk, N, K * d, generator=g)


def _masked_core(query, key, value, K, d):
    """The reference's masked temporal attention with its (Tq, Tk) mask broadcast over every problem: the reference itself raises
    for K != d (its mask.repeat(K B, ...) meets d B problems), the kernels take any K and d."""
    B = query.shape[0]
    q, k, v = (torch.cat(torch.split(t, K, dim=-1), dim=0).permute(0, 2, 1, 3) for t in (query, key, value))
    att = q @ k.transpose(-1, -2) / d ** 0.5
    keep = torch.ones(att.shape[-2:], dtype=torch.bool, device=att.device).tril()
    att = torch.where(keep, att, torch.tensor([G.MASKED_LOGIT], dtype=torch.float32, device=att.device))
    X = (torch.softmax(att, dim=-1) @ v).permute(0, 2, 1, 3)
    return torch.cat(torch.split(X, B, dim=0), dim=-1)


def _attn(q, k, v, K, d, spatial, mask, want, route, dtype):
    """Output and the asked-for gradients of <Gout, attention(q, k, v)> on one route: "fused" or "op"."""
    leaves = [t.to(DEV, dtype).requires_grad_(w in want) for t, w in zip((q, k, v), "qkv")]
    grad = bool(want)
    with torch.set_grad_enabled(grad):
        if route == "fused":
            y = ops.gman_attention(*leaves, d, K, G._attention_scale(d), spatial, mask, grad)
        elif spatial:
            y = G.spatial_attention_core(*leaves, K, d)
        elif mask and K != d:
            y = _masked_core(*leaves, K, d)
        else:
            y = G.temporal_attention_core(*leaves, K, d, mask)
        got = {"o": y.detach()}
        if grad:
            Gout = torch.randn(y.shape, generator=torch.Generator().manual_seed(99)).to(DEV, dtype)
            gs = torch.autograd.grad(y, [t for t, w in zip(leaves, "qkv") if w in want], Gout)
            got.update({w: gg for w, gg in zip([w for w in "qkv" if w in want], gs)})
    return got


def _check(q, k, v, K, d, spatial, mask, want="qkv"):
    f = _attn(q, k, v, K, d, spatial, mask, want, "fused", torch.float32)
    o = _attn(q, k, v, K, d, spatial, mask, want, "op", torch.float32)
    w = _attn(q, k, v, K, d, spatial, mask, want, "op", torch.float64)
    assert set(f) == set(w) == set("o" + want)
    for key in w:
        _criterion(f[key], o[key], w[key], key)


@pytest.mark.parametrize("N", [1, 2, 63, 64, 65, 325, 1000, 4096])
def test_spatial_kernel_nodes(N):
    B, T, K, d = (2, 3, 8, 8) if N <= 1000 else (1, 1, 5, 2)
    _check(*_qkv(B, T, T, N, K, d, seed=N), K, d, True, False)


@pytest.mark.parametrize("width", range(1, 17))
def test_kernels_every_width(width):
    heads = (1, 3, 8)[width % 3]
    _check(*_qkv(2, 3, 3, 70, width, heads, seed=width), width, heads, True, False)
    _check(*_qkv(2, 9, 9, 5, width, heads, seed=width + 100), width, heads, False, width % 2 == 0)


@pytest.mark.parametrize("Lq,Lk", [(1, 1), (12, 12), (31, 31), (32, 32), (33, 33), (64, 64), (12, 10), (10, 12), (1, 64), (64, 1),
                                   (33, 31)])
@pytest.mark.parametrize("mask", [False, True])
def test_short_kernel_lengths(Lq, Lk, mask):
    if mask and Lq != Lk:
        pytest.skip("the temporal mask is square (a transform attention has no mask)")
    _check(*_qkv(2, Lq, Lk, 7, 8, 3, seed=Lq * 100 + Lk), 8, 3, False, mask)


def test_sequences_past_64_run_op_for_op():
    m = G.TemporalAttention(3, 3, 0.1, True).to(DEV)
    X = torch.randn(2, 65, 5, 9, device=DEV)
    with _counted() as c:
        m(X, X).sum().backward()
        with torch.no_grad():
            m(X[:, :64], X[:, :64])
    assert _ran(c) == {"k_gman_attn_short_fwd": 1}, c
    assert not G.fused_route(torch.float32, True, 2, 65, 65, 5, 4, 2, "temporal", True, False, True)


@pytest.mark.parametrize("spatial,mask", [(True, False), (False, False), (False, True)])
def test_large_signed_logits(spatial, mask):
    q, k, v = _qkv(2, 12, 12, 40, 8, 3, seed=5, amp=6.0)      # |logits| well past 80, both signs
    assert float((q[0, 0, :, :8] @ k[0, 0, :, :8].T).abs().max()) / 3 ** 0.5 > 80
    _check(q, k, v, 8, 3, spatial, mask)


@pytest.mark.parametrize("want", ["q", "k", "v", "qk", "qv", "kv", "qkv"])
@pytest.mark.parametrize("spatial,mask", [(True, False), (False, True)])
def test_gradient_subsets(want, spatial, mask):
    _check(*_qkv(2, 6, 6, 33, 4, 4, seed=len(want)), 4, 4, spatial, mask, want)


# ---- determinism, equivariance, launch counts -----------------------------------------------------------------------------------------
def _pems_like(B=4, N=60, L=1, mask=True):
    c = dict(CASES["unit_l1"], B=B, N=N, L=L, mask=mask)
    return c, model_for(c, GMAN, DEV, torch.float32)


def test_training_forward_equals_no_grad_and_backward_repeats():
    c, m = _pems_like()
    from gman_seq import inputs, spatial_embedding
    X, TE, Gw = (t.to(DEV) for t in inputs(c, 0))
    SE = spatial_embedding(c).to(DEV)
    m.eval()                                  # running statistics: the FC / BatchNorm layers see the same numbers on every call
    with torch.no_grad():
        inf = m(X, SE, TE)
    outs, grads = [], []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        y = m(X, SE, TE)
        (y * Gw).sum().backward()
        outs.append(y.detach())
        grads.append({k: p.grad.clone() for k, p in m.named_parameters()})
    assert torch.equal(outs[0], inf) and torch.equal(outs[1], inf)
    assert all(torch.equal(grads[0][k], grads[1][k]) for k in grads[0])
    for e in (-3, 5):                         # loss scaled by 2^e: every gradient scales exactly
        m.zero_grad(set_to_none=True)
        (m(X, SE, TE) * Gw * 2.0 ** e).sum().backward()
        for k, p in m.named_parameters():
            assert torch.equal(p.grad, grads[0][k] * 2.0 ** e), k


def test_attention_bit_repeatable_and_scale_equivariant():
    q, k, v = (t.to(DEV).requires_grad_(True) for t in _qkv(3, 12, 12, 325, 8, 8, seed=1))
    for spatial, mask in ((True, False), (False, True)):
        with torch.no_grad():
            inf = ops.gman_attention(q, k, v, 8, 8, G._attention_scale(8), spatial, mask, False)
        gs = []
        for s in (1.0, 1.0, 8.0):
            y = ops.gman_attention(q, k, v, 8, 8, G._attention_scale(8), spatial, mask, True)
            assert torch.equal(y.detach(), inf)
            gs.append(torch.autograd.grad((y * s).sum(), (q, k, v)))
        assert all(torch.equal(a, b) for a, b in zip(gs[0], gs[1]))
        assert all(torch.equal(a * 8, b) for a, b in zip(gs[0], gs[2]))


def test_launch_counts():
    q, k, v = (t.to(DEV).requires_grad_(True) for t in _qkv(2, 12, 12, 50, 8, 8, seed=2))
    sc = G._attention_scale(8)
    for spatial, fwd, bwd in ((True, {"k_gman_attn_long_fwd": 1}, {"k_gman_attn_long_bwd_q": 1, "k_gman_attn_long_bwd_kv": 1}),
                              (False, {"k_gman_attn_short_fwd": 1}, {"k_gman_attn_short_bwd": 1})):
        with torch.no_grad(), _counted() as c:
            ops.gman_attention(q, k, v, 8, 8, sc, spatial, not spatial, False)
        assert _ran(c) == fwd
        y = ops.gman_attention(q, k, v, 8, 8, sc, spatial, not spatial, True)
        with _counted() as c:
            torch.autograd.grad(y.sum(), (q, k, v))
        assert _ran(c) == bwd
        if spatial:                            # dQ alone: the D pass only; dV alone: both passes
            y = ops.gman_attention(q, k.detach(), v.detach(), 8, 8, sc, True, False, True)
            with _counted() as c:
                torch.autograd.grad(y.sum(), q)
            assert _ran(c) == {"k_gman_attn_long_bwd_q": 1}
    for L in (1, 2):
        c_, m = _pems_like(B=2, N=20, L=L)
        from gman_seq import inputs, spatial_embedding
        X, TE, _ = (t.to(DEV) for t in inputs(c_, 0))
        with _counted() as c:
            y = m(X, spatial_embedding(c_).to(DEV), TE)
        assert _ran(c) == {"k_gman_attn_long_fwd": 2 * L, "k_gman_attn_short_fwd": 2 * L + 1}
        with _counted() as c:
            y.sum().backward()
        assert _ran(c) == {"k_gman_attn_long_bwd_q": 2 * L, "k_gman_attn_long_bwd_kv": 2 * L, "k_gman_attn_short_bwd": 2 * L + 1}


def test_spatial_attention_peak_memory_pems_bay():
    """One spatial attention's training forward at the PEMS-BAY shape (B = 16, 12 steps, N = 325, 8 heads of width 8): the op-for-op
    route allocates the 649 MB score tensor (and more); the fused route allocates O and the 0.8 MB stash."""
    q, k, v = (t.to(DEV).requires_grad_(True) for t in _qkv(16, 12, 12, 325, 8, 8, seed=3))
    score_bytes = 16 * 12 * 8 * 325 * 325 * 4
    peaks = {}
    for route in ("fused", "op"):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        y = ops.gman_attention(q, k, v, 8, 8, G._attention_scale(8), True, False, True) if route == "fused" else \
            G.spatial_attention_core(q, k, v, 8, 8)
        torch.cuda.synchronize()
        peaks[route] = torch.cuda.max_memory_allocated() - base
        del y
    assert peaks["op"] >= score_bytes, peaks
    assert peaks["fused"] <= q.numel() * 4 + 16 * 12 * 8 * 325 * 4 + (1 << 20), peaks
    assert peaks["fused"] * 20 < score_bytes, peaks


def test_cuda_graph_training_step():
    """A whole training step (forward, MAE, backward, capturable Adam) captured once and replayed, against the same steps run eagerly."""
    c, m = _pems_like(B=4, N=30, L=1, mask=True)
    from gman_seq import inputs, spatial_embedding
    X, TE, _ = (t.to(DEV) for t in inputs(c, 0))
    Y = torch.rand(c["B"], c["pred"], c["N"], device=DEV)
    SE = spatial_embedding(c).to(DEV)
    eager = copy.deepcopy(m)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)
    opt_e = torch.optim.Adam(eager.parameters(), lr=1e-3, capturable=True)

    def step(model, o):
        o.zero_grad(set_to_none=False)
        loss = (model(X, SE, TE) - Y).abs().mean()
        loss.backward()
        o.step()
        return loss

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(m, opt)
            step(eager, opt_e)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with _counted() as cnt, torch.cuda.graph(g):
        static_loss = step(m, opt)
    assert _ran(cnt).get("k_gman_attn_long_bwd_kv") == 2, cnt
    losses = []
    for _ in range(3):
        g.replay()
        losses.append(static_loss.clone())
        le = step(eager, opt_e)
        torch.testing.assert_close(losses[-1], le, rtol=1e-5, atol=1e-6)
    torch.cuda.synchronize()
    assert losses[0] != losses[2]
    for (k, p), pe in zip(m.named_parameters(), eager.parameters()):
        torch.testing.assert_close(p, pe, rtol=1e-4, atol=1e-5, msg=k)


# ---- routing and the ABI ---------------------------------------------------------------------------------------------------------------
def test_routes_outside_the_envelope_run_op_for_op():
    X = torch.rand(2, 4, 9, device=DEV)
    SE = torch.randn(9, 34, device=DEV)
    TE = torch.zeros(2, 7, 2, device=DEV)
    for m, args in ((GMAN(1, 17, 2, 4, 0.1, 12, True, False), (X, SE, TE)),           # head width 17
                    (GMAN(1, 2, 17, 4, 0.1, 12, True, False).double(), (X.double(), SE.double(), TE))):
        m = m.to(DEV)
        with _counted() as c:
            m(*args).sum().backward()
        assert _ran(c) == {}, c
    m = GMAN(1, 4, 4, 4, 0.1, 12, True, True).to(DEV)
    m.fused_training = False
    with _counted() as c:
        m(X, torch.randn(9, 16, device=DEV), TE).sum().backward()
    assert _ran(c) == {}
    with pytest.raises(RuntimeError, match="must match the size"):
        GMAN(1, 4, 8, 4, 0.1, 12, True, True).to(DEV)(X, torch.randn(9, 32, device=DEV), TE)


def test_abi_errors():
    L_ = _lib.lib()
    assert L_.stmp_gman_attn_supported(2, 3, 8, 8, 325, 325, 0, 1) == 1
    assert L_.stmp_gman_attn_supported(2, 3, 8, 17, 325, 325, 0, 1) == 0          # width
    assert L_.stmp_gman_attn_supported(2, 3, 8, 8, 12, 12, 1, 1) == 0             # the long kernel has no mask
    assert L_.stmp_gman_attn_supported(2, 3, 8, 8, 65, 12, 0, 0) == 0             # short: Lq, Lk <= 64
    assert L_.stmp_gman_attn_supported(2, 3, 8, 8, 12, 10, 1, 0) == 0             # a mask is square
    assert L_.stmp_gman_attn_supported(1 << 30, 1 << 10, 8, 8, 12, 12, 0, 0) == 0 # grid
    assert L_.stmp_gman_attn_supported(0, 3, 8, 8, 12, 12, 0, 0) == 1
    q = torch.zeros(2, 12, 5, 8, device=DEV)
    strides = (ctypes.c_int64 * 12)(*([q.stride(0), q.stride(2), q.stride(1)] * 4))
    p = _lib.ptr(q)
    with _counted() as c:
        rc = L_.stmp_gman_attn_fwd(2, 5, 1, 17, 12, 12, 0, 0, 1.0, strides, p, p, p, p, None, _lib.stream_ptr())
        assert rc == _lib.STMP_EUNSUPPORTED and "outside the envelope" in _lib.last_error()
        rc = L_.stmp_gman_attn_fwd(2, 5, 1, 8, 12, 12, 0, 0, 1.0, None, p, p, p, p, None, _lib.stream_ptr())
        assert rc == _lib.STMP_EINVAL
        rc = L_.stmp_gman_attn_fwd(-1, 5, 1, 8, 12, 12, 0, 0, 1.0, strides, p, p, p, p, None, _lib.stream_ptr())
        assert rc == _lib.STMP_EINVAL
        rc = L_.stmp_gman_attn_bwd(2, 5, 1, 8, 12, 12, 0, 0, 1.0, strides, p, p, p, p, None, p, None, p, None, None,
                                   _lib.stream_ptr())
        assert rc == _lib.STMP_EINVAL and "stash" in _lib.last_error()
        assert L_.stmp_gman_attn_fwd(0, 5, 1, 8, 12, 12, 0, 0, 1.0, strides, None, None, None, None, None, _lib.stream_ptr()) == 0
        empty = torch.zeros(0, 12, 5, 8, device=DEV, requires_grad=True)
        y = ops.gman_attention(empty, empty, empty, 1, 8, 1.0, False, False, True)
        y.sum().backward()
    assert _ran(c) == {}, c
    with pytest.raises(RuntimeError, match="gman_attention"):
        ops.gman_attn_fwd(q, q[:, :3, :4], q[:, :3, :4], 1, 8, 1.0, True, False)
