"""GMAN without a GPU: the op-for-op restatement against the unmodified reference (every golden case: training steps, running
statistics, gradients, the eval call), its attention cores bit for bit, the fused attention backward's algebra (gman_attention.cu's decomposition, in float64
torch) against autograd, the state_dict keys and seeded initialisation against the reference's, the reference's K != d mask error,
the routing predicate and the refusal of CPU tensors."""
import pytest
import torch

from gman_seq import CASES, build, cpu_batchnorm_fix, model_for, run
from oracle import refload
from pytorch_geometric_temporal_b200.nn.attention import GMAN, SpatioTemporalAttention, SpatioTemporalEmbedding
from pytorch_geometric_temporal_b200.nn.attention import gman as G

D = torch.float64


def _ref_module():
    if not refload.available():
        pytest.skip("reference tree not present")
    return refload.load("nn.attention.gman")


@pytest.fixture
def on_cpu(monkeypatch):
    """Lift the modules' CUDA-only check so the op-for-op route runs on CPU tensors."""
    monkeypatch.setattr(G, "_require_cuda", lambda t, name: None)


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_reference(name, on_cpu):
    """The whole model, op for op on CPU in float64, against the reference: every output, cost, running statistic and gradient.  The
    1 x 1 convolutions run as F.linear, which sums in another order than the reference's conv2d, so agreement is to 1e-11 of each
    tensor's scale; a conv bias in front of a BatchNorm has a gradient that is zero in exact arithmetic, a cancellation of terms as
    large as the run's largest gradient, so gradients also get 1e-9 of that."""
    ref_mod = _ref_module()
    c = CASES[name]
    old = torch.get_default_dtype()
    torch.set_default_dtype(D)               # the reference builds its one-hot in the default dtype
    try:
        with cpu_batchnorm_fix():
            want = run(model_for(c, ref_mod.GMAN, "cpu", D), c, "cpu", D)
        got = run(model_for(c, GMAN, "cpu", D), c, "cpu", D)
    finally:
        torch.set_default_dtype(old)
    assert set(got) == set(want)
    gscale = max(float(v.abs().max()) for k, v in want.items() if k.startswith("grad."))
    for k in want:
        assert got[k].dtype == want[k].dtype, k
        if want[k].dtype == torch.int64:
            assert torch.equal(got[k], want[k]), k
            continue
        tol = 1e-11 * float(want[k].abs().max()) + (1e-9 * gscale if k.startswith("grad.") else 0.0)
        assert float((got[k] - want[k]).abs().max()) <= tol, (k, float((got[k] - want[k]).abs().max()), tol)


@pytest.mark.parametrize("K,d,mask", [(8, 8, False), (4, 16, False), (16, 4, False), (4, 2, True), (2, 5, False)])
def test_attention_cores_match_reference_bit_for_bit(K, d, mask):
    """The op-for-op attention cores against the reference's attentions with their FullyConnected layers replaced by identities (so
    Q = K = V = [X | STE], 2 d heads of width K, the reference's 1/sqrt(d) scaling; with the mask K = 2 d, so the reference's mask
    broadcasts): equal bit for bit, forward and backward."""
    ref_mod = _ref_module()
    g = torch.Generator().manual_seed(3)
    B, T, N = 3, 5, 7
    X = torch.randn(B, T, N, K * d, generator=g, dtype=D, requires_grad=True)
    STE = torch.randn(B, T, N, K * d, generator=g, dtype=D, requires_grad=True)
    STE_pred = torch.randn(B, T + 2, N, K * d, generator=g, dtype=D, requires_grad=True)
    sp = ref_mod.SpatialAttention(K, d, 0.1)
    tm = ref_mod.TemporalAttention(K, d, 0.1, mask) if mask else ref_mod.TemporalAttention(K, d, 0.1, False)
    tr = ref_mod.TransformAttention(K, d, 0.1)
    for m in (sp, tm, tr):
        for n in ("_fully_connected_q", "_fully_connected_k", "_fully_connected_v", "_fully_connected"):
            setattr(m, n, torch.nn.Identity())
    XS = torch.cat((X, STE), dim=-1)
    pairs = [(sp(X, STE), G.spatial_attention_core(XS, XS, XS, K, d)),
             (tm(X, STE), G.temporal_attention_core(XS, XS, XS, K, d, mask)),
             (tr(X, STE, STE_pred), G.temporal_attention_core(STE_pred, STE, X, K, d, False))]
    for want, got in pairs:
        assert torch.equal(got, want)
        gw = torch.autograd.grad(want, (X, STE), torch.ones_like(want), allow_unused=True)
        gg = torch.autograd.grad(got, (X, STE), torch.ones_like(got), allow_unused=True)
        assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(gw, gg))


def _heads(t, K):
    """(B, T, N, K d) -> (d, B, T, N, K): head h = channels [h K, (h + 1) K)."""
    return torch.stack(torch.split(t, K, dim=-1))


def hand_attention_backward(q, k, v, K, d, spatial, mask, g):
    """gman_attention.cu's forward and backward in float64 torch, per (problem, head): logits S = scale Q K^T (masked logits -32767),
    lse = logsumexp(S), O = exp(S - lse) V; then D = rowsum(dO . O), P recomputed from lse, dS = P (dO V^T - D) with the masked entries
    zeroed, dQ = scale dS K, dK = scale dS^T Q, dV = P^T dO."""
    scale = 1.0 / d ** 0.5
    Q, Kt, V, Gh = (_heads(t, K) for t in (q, k, v, g))
    if not spatial:                          # attend over the steps: (d, B, N, T, K)
        Q, Kt, V, Gh = (t.transpose(2, 3) for t in (Q, Kt, V, Gh))
    S = scale * Q @ Kt.transpose(-1, -2)
    keep = torch.ones(S.shape[-2:], dtype=torch.bool).tril() if mask else torch.ones(S.shape[-2:], dtype=torch.bool)
    S = torch.where(keep, S, torch.tensor(float(G.MASKED_LOGIT), dtype=D))
    lse = torch.logsumexp(S, dim=-1, keepdim=True)
    O = torch.exp(S - lse) @ V
    Dl = (Gh * O).sum(-1, keepdim=True)
    P = torch.exp(S - lse)
    dS = torch.where(keep, P * (Gh @ V.transpose(-1, -2) - Dl), torch.zeros((), dtype=D))
    dQ, dK, dV = scale * dS @ Kt, scale * dS.transpose(-1, -2) @ Q, P.transpose(-1, -2) @ Gh

    def back(t):
        if not spatial:
            t = t.transpose(2, 3)
        return torch.cat(tuple(t), dim=-1)
    return back(O), back(dQ), back(dK), back(dV)


@pytest.mark.parametrize("spatial,mask,K,d,Tq,Tk", [(True, False, 8, 8, 5, 5), (True, False, 4, 3, 3, 3), (False, False, 4, 3, 7, 7),
                                                    (False, True, 3, 3, 7, 7), (False, False, 5, 2, 4, 9), (False, True, 1, 1, 1, 1)])
def test_attention_backward_algebra(spatial, mask, K, d, Tq, Tk):
    g = torch.Generator().manual_seed(7)
    B, N = 2, 6
    Dm = K * d
    q = (torch.randn(B, Tq, N, Dm, generator=g, dtype=D) * 3).requires_grad_(True)
    k = (torch.randn(B, Tk if not spatial else Tq, N, Dm, generator=g, dtype=D) * 3).requires_grad_(True)
    v = torch.randn(k.shape, generator=g, dtype=D).requires_grad_(True)
    out = G.spatial_attention_core(q, k, v, K, d) if spatial else G.temporal_attention_core(q, k, v, K, d, mask)
    gout = torch.randn(out.shape, generator=g, dtype=D)
    want = torch.autograd.grad(out, (q, k, v), gout)
    O, dQ, dK, dV = hand_attention_backward(q.detach(), k.detach(), v.detach(), K, d, spatial, mask, gout)
    assert torch.allclose(O, out.detach(), rtol=1e-12, atol=1e-12)
    for got, w, n in zip((dQ, dK, dV), want, "qkv"):
        assert torch.allclose(got, w, rtol=1e-10, atol=1e-12), n
    if mask:                                 # masked logits get no gradient: dQ of row 0 sees only key 0
        qs = q.detach().clone().requires_grad_(True)
        o0 = G.temporal_attention_core(qs, k.detach(), v.detach(), K, d, True)[:, 0]
        gq, = torch.autograd.grad(o0, qs, torch.ones_like(o0))
        assert torch.equal(gq[:, 1:], torch.zeros_like(gq[:, 1:]))


def test_state_dict_and_seeded_init_match_reference():
    ref_mod = _ref_module()
    for args in ((1, 8, 8, 12, 0.1, 288, True, False), (2, 4, 16, 6, None, 24, False, True)):
        torch.manual_seed(11)
        ref = ref_mod.GMAN(*args)
        torch.manual_seed(11)
        ours = GMAN(*args)
        sr, so = ref.state_dict(), ours.state_dict()
        assert list(sr) == list(so)
        for k in sr:
            assert torch.equal(sr[k], so[k]), k
        assert "_st_att_block1.0._spatial_attention._fully_connected_q._conv2ds.0._conv2d.weight" in so
        assert sum(1 for m in ours.modules() if isinstance(m, torch.nn.BatchNorm2d)) == 12 + 24 * args[0]     # 36 at L = 1
        ours2 = GMAN(*args)
        ours2.load_state_dict(sr)
    for cls, args in ((SpatioTemporalEmbedding, (16, 0.1, 24, False)), (SpatioTemporalAttention, (4, 4, 0.1, True))):
        torch.manual_seed(5)
        r = getattr(ref_mod, cls.__name__)(*args).state_dict()
        torch.manual_seed(5)
        o = cls(*args).state_dict()
        assert list(r) == list(o) and all(torch.equal(r[k], o[k]) for k in r)


def test_mask_with_k_not_d_raises_like_reference(on_cpu):
    ref_mod = _ref_module()
    c = dict(CASES["k4_d16"], mask=True)
    X = torch.rand(2, c["his"], c["N"])
    SE = torch.randn(c["N"], 64)
    TE = torch.zeros(2, c["his"] + c["pred"], 2)
    torch.manual_seed(0)
    with pytest.raises(RuntimeError):
        build(ref_mod.GMAN, c)(X, SE, TE)
    ours = build(GMAN, c)
    before = {k: v.clone() for k, v in ours.state_dict().items()}
    with pytest.raises(RuntimeError, match="must match the size"):
        ours(X, SE, TE)
    assert all(torch.equal(before[k], v) for k, v in ours.state_dict().items())     # raised before any layer ran
    G.check_mask(1, 4, 1, True)              # a one-problem mask broadcasts in the reference: no error
    G.check_mask(4, 4, 3, True)
    G.check_mask(4, 16, 3, False)


def test_routing_predicate():
    f32, f64 = torch.float32, torch.float64
    base = dict(dtype=f32, is_cuda=True, batch=16, Lq=12, Lk=12, other=325, K=8, d=8, kind="temporal", mask=True, needs_grad=True,
                fused_training=True)

    def route(**kw):
        return G.fused_route(**dict(base, **kw))
    assert route()
    assert route(kind="transform", Lq=12, Lk=64, mask=False)
    assert route(kind="spatial", Lq=4096, Lk=4096, other=12, mask=False)
    assert route(K=16) and route(K=1) and not route(K=17)
    assert not route(dtype=f64) and not route(is_cuda=False)
    assert not route(Lq=65, Lk=65) and not route(kind="transform", Lq=12, Lk=65, mask=False)
    assert not route(fused_training=False) and route(fused_training=False, needs_grad=False)
    assert route(batch=0)


def test_modules_refuse_cpu_tensors():
    m = GMAN(1, 2, 2, 3, 0.1, 12, True, False)
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.rand(2, 3, 5), torch.randn(5, 4), torch.zeros(2, 5, 2))
    with pytest.raises(RuntimeError, match="CUDA only"):
        SpatioTemporalAttention(2, 2, 0.1, False)(torch.rand(2, 3, 5, 4), torch.rand(2, 3, 5, 4))
    with pytest.raises(RuntimeError, match="CUDA only"):
        SpatioTemporalEmbedding(4, 0.1, 12)(torch.randn(5, 4), torch.zeros(2, 5, 2), 12)


def test_fused_training_switch_reaches_every_attention():
    m = GMAN(2, 2, 2, 3, 0.1, 12, True, False)
    assert m.fused_training
    m.fused_training = False
    atts = [a for a in m.modules() if isinstance(a, G._Attention)]
    assert len(atts) == 9 and not any(a._fused for a in atts) and not m._st_att_block1[0].fused_training
    m._st_att_block2[1].fused_training = True
    assert not m.fused_training and m._st_att_block2[1].fused_training
