"""AGCRN on the H100: every golden case on both routes (the fused kernels and op for op) against the reference's float64 values, the
envelope against a float64 run of the op-for-op algebra, adversarial embeddings (logits past 80, all-zero rows, exact e_n . e_m = 0
kinks), bit-reproducible calls and backwards, the training forward against the no_grad call, loss-scale equivariance, retain_graph,
CUDA-graph replay of the tutorial epoch, exact launch counts, the routes outside the envelope and the ABI's errors.

The criterion, per tensor (DESIGN §5): the fused route's largest error against float64 is at most 4 times the float32 op-for-op route's
plus 2^-20 of the tensor's largest float64 magnitude.  Goldens of more than 16 384 elements are held to the same criterion through
their fingerprints (four fixed projections and the norm), with the norm as the scale."""
import ctypes
import os

import pytest
import torch

from agcrn_seq import CASES, fingerprint, inputs, load, model_for, run
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import AGCRN
from pytorch_geometric_temporal_b200.nn.recurrent.agcrn import agcrn_cell
from test_gpu_rows_envelope import _counted

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FWD = ("k_agcrn_support", "k_agcrn_gemm_nodew", "k_agcrn_gemm_sup_gate", "k_agcrn_gemm_con_gate", "k_agcrn_gemm_sup_update",
       "k_agcrn_gemm_con_update")
BWD = ("k_agcrn_pw_update", "k_agcrn_gemm_df_update", "k_agcrn_gemm_dw_update", "k_agcrn_gemm_supt_update", "k_agcrn_pw_gate",
       "k_agcrn_gemm_dw_gate", "k_agcrn_gemm_df_gate", "k_agcrn_gemm_supt_gate", "k_agcrn_gemm_dpool")
EGRAD = ("k_agcrn_gemm_dt", "k_agcrn_softmax_bwd", "k_agcrn_gemm_de")
ALL = FWD + BWD + EGRAD + ("k_agcrn_gemm_t2", "k_agcrn_gemm_ds", "k_agcrn_split_reduce_dt", "k_agcrn_split_reduce_de")


@pytest.fixture(autouse=True)
def _fp32():
    """cuBLAS in full fp32 on the op-for-op route."""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


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
    m = model_for(c, AGCRN, DEV, torch.float32)
    for layer in m.layers:
        layer.fused_training = fused
    with _counted() as cnt:
        out, cost, grads = run(m, c, DEV, torch.float32)
    torch.cuda.synchronize()
    return out, cost, grads, _ran(cnt)


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_both_routes(name):
    c = load(GOLDEN)["cases"][name]
    of, cf, gf, ran_f = _run_route(CASES[name], True)
    oo, co, go, ran_o = _run_route(CASES[name], False)
    assert ran_o == {} and set(ran_f) >= set(FWD + BWD), (ran_o, ran_f)
    got_f = dict(out=of, **{f"grad.{k}": v for k, v in gf.items()})
    got_o = dict(out=oo, **{f"grad.{k}": v for k, v in go.items()})
    assert set(got_f) == set(c["fingerprints"]), (sorted(got_f), sorted(c["fingerprints"]))
    _criterion(cf.view(1), co.view(1), c["cost"].view(1), "cost")
    for k, fp in c["fingerprints"].items():
        if k in c["values"]:
            _criterion(got_f[k], got_o[k], c["values"][k].double(), k)
        else:
            _criterion(fingerprint(got_f[k]), fingerprint(got_o[k]), fp, k, scale=float(fp[-1]))


# ---- the envelope against float64 -----------------------------------------------------------------------------------------------------
# (K, in, out, d, N, B, H given, gradients asked for: x / h / e / pools)
ENVELOPE = [
    (1, 8, 2, 4, 20, 1, False, "xep"), (2, 8, 2, 4, 20, 3, True, "xhep"), (3, 8, 2, 4, 20, 3, True, "xhep"),
    (1, 1, 1, 1, 1, 1, True, "xhep"), (2, 127, 1, 1, 1, 3, True, "xh"), (3, 1, 1, 64, 2, 64, False, "p"),
    (2, 64, 16, 32, 100, 1, True, "xhep"), (3, 64, 16, 32, 100, 3, True, "e"), (1, 64, 16, 32, 100, 3, False, "x"),
    (2, 96, 31, 10, 63, 3, True, "hp"), (3, 96, 32, 10, 64, 3, True, "xhep"), (1, 95, 33, 10, 65, 3, True, "xhep"),
    (2, 64, 64, 10, 127, 3, True, "xhep"), (3, 64, 64, 64, 128, 1, True, "xhep"), (1, 64, 64, 10, 129, 3, False, "ep"),
    (2, 1, 64, 10, 307, 64, True, "xhep"), (2, 16, 2, 4, 191, 0, True, "xhep"), (3, 5, 33, 4, 192, 3, True, ""),
    (2, 3, 16, 4, 193, 64, False, "xep"), (2, 1, 64, 10, 4096, 1, True, "xhep"), (3, 64, 64, 10, 4096, 1, False, "p"),
    (1, 32, 32, 64, 4095, 3, True, "xh"), (2, 112, 16, 4, 1000, 3, True, "xhep"), (3, 120, 2, 32, 255, 64, False, "xep"),
]


def _float64_case(K, cin, out, d, N, B, with_h, want, seed, embed=None):
    """(inputs, parameters) of one envelope call: float32 values, E scaled so the logits stay O(1) unless `embed` supplies E."""
    g = torch.Generator().manual_seed(seed)
    f32 = dict(generator=g, dtype=torch.float32)
    X = torch.randn(B, N, cin, **f32)
    E = torch.randn(N, d, **f32) / d ** 0.5 if embed is None else embed
    H = torch.randn(B, N, out, **f32) if with_h else None
    pools = [torch.randn(d, K, cin + out, 2 * out, **f32) / (cin + out) ** 0.5, torch.randn(d, 2 * out, **f32) * 0.3,
             torch.randn(d, K, cin + out, out, **f32) / (cin + out) ** 0.5, torch.randn(d, out, **f32) * 0.3]
    return X, E, H, pools


def _eval(X, E, H, pools, K, out, want, fused, dtype):
    """Output and the asked-for gradients of <G, AGCRN(X, E, H)> for a fixed random G on one route."""
    leaves = [None if t is None else t.to(DEV, dtype).requires_grad_(w) for t, w in
              ((X, "x" in want), (E, "e" in want), (H, "h" in want))]
    ps = [p.to(DEV, dtype).requires_grad_("p" in want) for p in pools]
    grad = bool(want) and (("x" in want) or ("e" in want) or ("h" in want and H is not None) or "p" in want)
    with torch.set_grad_enabled(grad):
        y = ops.agcrn_train(*leaves, *ps) if fused and grad else (ops.agcrn_fwd(*leaves, *ps) if fused else
                                                                   agcrn_cell(*leaves, (*ps[:2], K), (*ps[2:], K), out))
        G = torch.randn(y.shape, generator=torch.Generator().manual_seed(99)).to(DEV, dtype)
        got = {"y": y.detach()}
        if grad:
            (y * G).sum().backward()
            for name, t in zip(("x", "e", "h"), leaves):
                if t is not None and t.requires_grad:
                    got["d" + name] = t.grad
            if "p" in want:
                got.update({f"dp{i}": p.grad for i, p in enumerate(ps)})
    return got


def _check_three_ways(K, cin, out, d, N, B, with_h, want, seed, embed=None):
    X, E, H, pools = _float64_case(K, cin, out, d, N, B, with_h, want, seed, embed)
    ref = _eval(X, E, H, pools, K, out, want, False, torch.float64)
    op = _eval(X, E, H, pools, K, out, want, False, torch.float32)
    with _counted() as cnt:
        fu = _eval(X, E, H, pools, K, out, want, True, torch.float32)
    assert set(fu) == set(ref), (sorted(fu), sorted(ref))
    for k in ref:
        _criterion(fu[k], op[k], ref[k], (K, cin, out, d, N, B, with_h, want, k))
    return _ran(cnt)


@pytest.mark.parametrize("K,cin,out,d,N,B,with_h,want", ENVELOPE)
def test_envelope_against_float64(K, cin, out, d, N, B, with_h, want):
    ran = _check_three_ways(K, cin, out, d, N, B, with_h, want, seed=N + 7 * K + out)
    assert B == 0 and ran == {} or B > 0 and set(ran) >= set(FWD), ran


@pytest.mark.parametrize("kind", ["large_logits", "zero_rows", "kinks"])
def test_adversarial_embeddings(kind):
    N, d = 70, 8
    g = torch.Generator().manual_seed(4)
    if kind == "large_logits":               # self logits of 81 .. 144: exp without the max subtraction overflows
        E = torch.randn(N, d, generator=g)
        E = E / E.norm(dim=1, keepdim=True) * (9 + 3 * torch.rand(N, 1, generator=g))
    elif kind == "zero_rows":                # rows 0, 5, 10, ... embed to 0: all-zero logits, a uniform row of S
        E = torch.randn(N, d, generator=g)
        E[::5] = 0
    else:                                    # integer embeddings with many exact e_n . e_m = 0 (ReLU's kink, gradient 0 as torch's)
        E = torch.randint(-1, 2, (N, d), generator=g).float()
    assert E.dtype == torch.float32
    for K in (1, 2, 3):
        _check_three_ways(K, 6, 5, d, N, 3, True, "xhep", seed=K, embed=E)


# ---- determinism, the training forward, equivariance, retain_graph ----------------------------------------------------------------------
def _tutorial_model(K=2):
    c = dict(CASES["tutorial_e"], K=K)
    return model_for(c, AGCRN, DEV, torch.float32), c


@pytest.mark.parametrize("K", [1, 2, 3])
def test_training_forward_equals_no_grad_and_repeats(K):
    m, c = _tutorial_model(K)
    layer = m.layers[0]
    E, X, _ = (t.to(DEV) for t in inputs(c))
    H = torch.randn(1, 20, 2, device=DEV)
    with torch.no_grad():
        want = layer(X[5], E, H)
    grads = []
    for _ in range(2):
        m.zero_grad()
        e = E.clone().requires_grad_(True)
        h = H.clone().requires_grad_(True)
        y = layer(X[5], e, h)
        assert torch.equal(y.detach(), want)
        (y * torch.arange(40, device=DEV).view(1, 20, 2)).sum().backward()
        grads.append([t.grad.clone() for t in (e, h, *layer.parameters())])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def _tutorial_grads(scale, steps=10):
    """The gradients of E and the parameters of `scale` times the tutorial's cost over its first `steps` snapshots."""
    m, c = _tutorial_model(2)
    E, X, Y = (t.to(DEV) for t in inputs(c))
    E.requires_grad_(True)
    h, cost = None, 0
    for t in range(steps):
        h = m.layers[0](X[t], E, h)
        cost = cost + torch.mean((m.linear(torch.relu(h)) - Y[t].view(1, 20, 1)) ** 2)
    (cost * scale).backward()
    return [E.grad, *(p.grad for p in m.parameters())]


def test_loss_scale_equivariance_and_retain_graph():
    for a, b in zip(_tutorial_grads(1.0), _tutorial_grads(8.0)):
        assert torch.equal(b, 8 * a)
    m, c = _tutorial_model(2)
    E, X, _ = (t.to(DEV) for t in inputs(c))
    E.requires_grad_(True)
    h = m.layers[0](X[0], E)
    h = m.layers[0](X[1], E, h)
    loss = h.square().sum()
    loss.backward(retain_graph=True)
    first = [t.grad.clone() for t in (E, *m.layers.parameters())]
    loss.backward()
    for a, t in zip(first, (E, *m.layers.parameters())):
        assert torch.equal(t.grad, 2 * a)


# ---- CUDA graphs, launch counts, routing, ABI ---------------------------------------------------------------------------------------------
def _paper_model(fused, B):
    """The paper's two layers (1 -> 64, 64 -> 64, d = 10, K = 2) on 307 nodes with a trained E, Linear(64, 1), T = 12 steps of B windows,
    on one route; returns (params, step), step = zero_grad, forward, MSE, backward and a capturable Adam step."""
    torch.manual_seed(0)
    layers = [AGCRN(307, 1, 64, 2, 10).to(DEV), AGCRN(307, 64, 64, 2, 10).to(DEV)]
    for layer in layers:
        layer.fused_training = fused
    lin = torch.nn.Linear(64, 1).to(DEV)
    E = torch.nn.Parameter(torch.randn(307, 10, device=DEV))
    g = torch.Generator().manual_seed(1)
    X, Y = torch.randn(B, 12, 307, 1, generator=g).to(DEV), torch.randn(B, 307, 1, generator=g).to(DEV)
    h0 = torch.zeros(B, 307, 64, device=DEV)
    params = [E, *layers[0].parameters(), *layers[1].parameters(), *lin.parameters()]
    opt = torch.optim.Adam(params, lr=1e-3, capturable=True)

    def step():
        opt.zero_grad(set_to_none=False)
        h1 = h2 = h0
        for t in range(12):
            h1 = layers[0](X[:, t], E, h1)
            h2 = layers[1](h1, E, h2)
        torch.mean((lin(h2) - Y) ** 2).backward()
        opt.step()
    for p in params:
        p.grad = torch.zeros_like(p)
    return params, step


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "op_for_op"])
def test_cuda_graph_paper_training_step(fused):
    """The paper's training step captured whole (both layers, 12 steps, backward, capturable Adam) and replayed: the replay's gradients
    equal an eager step's from the same state, and the parameters move."""
    params, step = _paper_model(fused, 16)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    before = [p.detach().clone() for p in params]
    graph.replay()
    torch.cuda.synchronize()
    got = [p.grad.clone() for p in params]
    ref_params, ref_step = _paper_model(fused, 16)
    with torch.no_grad():
        for p, b in zip(ref_params, before):
            p.copy_(b)
    ref_step()
    torch.cuda.synchronize()
    for i, (a, p) in enumerate(zip(got, ref_params)):
        if fused:
            assert torch.equal(a, p.grad), i
        else:
            assert torch.allclose(a, p.grad, rtol=1e-4, atol=1e-6 * float(p.grad.abs().max())), i
    assert any(not torch.equal(p.detach(), b) for p, b in zip(params, before))


def test_cuda_graph_tutorial_epoch():
    m, c = _tutorial_model(2)
    E, X, Y = (t.to(DEV) for t in inputs(c))
    E.requires_grad_(True)
    layer, lin = m.layers[0], m.linear

    def epoch():
        h, cost = None, 0
        for t in range(X.shape[0]):
            h = layer(X[t], E, h)
            cost = cost + torch.mean((lin(torch.relu(h)) - Y[t].view(1, 20, 1)) ** 2)
        cost = cost / X.shape[0]
        cost.backward()
        return cost

    params = [E, *m.parameters()]
    want = epoch().detach()
    want_g = [p.grad.clone() for p in params]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for p in params:
            p.grad = None
        epoch()
    torch.cuda.current_stream().wait_stream(s)
    for p in params:
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = epoch()
    for p in params:
        p.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(got.detach(), want)
    for p, w in zip(params, want_g):
        assert torch.equal(p.grad, w)


@pytest.mark.parametrize("K", [1, 2, 3])
def test_launch_counts(K):
    m = AGCRN(30, 4, 8, K, 5).to(DEV)
    X, E, H = torch.randn(3, 30, 4, device=DEV), torch.randn(30, 5, device=DEV), torch.randn(3, 30, 8, device=DEV)
    fwd = {k: 1 for k in FWD}
    if K == 3:
        fwd["k_agcrn_gemm_t2"] = 1
    with torch.no_grad(), _counted() as cnt:
        m(X, E, H)
    assert _ran(cnt) == fwd
    with _counted() as cnt:                  # pools only: no dF / transposed support product for the gate, no dE
        m(X, E, H).sum().backward()
    want = dict(fwd, **{k: 1 for k in BWD if k not in ("k_agcrn_gemm_df_gate", "k_agcrn_gemm_supt_gate")})
    assert _ran(cnt) == want
    with _counted() as cnt:
        m(X.requires_grad_(), E.requires_grad_(), H.requires_grad_()).sum().backward()
    want = dict(fwd, **{k: 1 for k in BWD + EGRAD})
    if K == 3:
        want["k_agcrn_gemm_ds"] = 1
    assert _ran(cnt) == want
    with torch.no_grad(), _counted() as cnt:   # B = 0: no launch
        assert m(X[:0], E).shape == (0, 30, 8)
    assert _ran(cnt) == {}


@pytest.mark.parametrize("what", ["float64", "K4", "out65", "in_plus_out129", "d65", "N4097", "no_fused_training"])
def test_routes_outside_envelope_op_for_op(what):
    shape = dict(K4=(10, 3, 4, 4, 3), out65=(10, 2, 65, 2, 3), in_plus_out129=(10, 65, 64, 2, 3), d65=(10, 3, 4, 2, 65),
                 N4097=(4097, 1, 2, 2, 3)).get(what, (10, 3, 4, 2, 3))
    N, cin, out, K, d = shape
    dtype = torch.float64 if what == "float64" else torch.float32
    torch.manual_seed(0)
    m = AGCRN(*shape).to(DEV, dtype)
    m.fused_training = what != "no_fused_training"
    X, E = torch.randn(2, N, cin, device=DEV, dtype=dtype), torch.randn(N, d, device=DEV, dtype=dtype).requires_grad_()
    with _counted() as cnt:
        y = m(X, E)
        y.sum().backward()
    assert _ran(cnt) == {}, cnt
    gate, update = ((a.detach().double(), b.detach().double(), K) for a, b in ((m._gate.weights_pool, m._gate.bias_pool),
                                                                               (m._update.weights_pool, m._update.bias_pool)))
    want = agcrn_cell(X.double(), E.detach().double(), None, gate, update, out)
    assert torch.allclose(y.detach().double(), want, rtol=1e-4, atol=1e-5)


def test_abi_errors():
    L = _lib.lib()
    buf = torch.zeros(3, 1 << 14, device=DEV)
    p, scr, hout = (ctypes.c_void_p(t.data_ptr()) for t in buf)     # inputs, scratch, output
    st = _lib.stream_ptr()

    def fwd(b=2, n=10, cin=3, out=4, K=2, d=5, x=p, e=p, scratch=scr):
        return L.stmp_agcrn_fwd(b, n, cin, out, K, d, x, e, None, p, p, p, p, scratch, None, hout, st)

    assert fwd() == _lib.STMP_OK
    assert fwd(x=None) == _lib.STMP_EINVAL
    assert fwd(e=None) == _lib.STMP_EINVAL
    assert fwd(scratch=None) == _lib.STMP_EINVAL
    assert fwd(b=-1) == _lib.STMP_EINVAL
    assert fwd(b=0, x=None, scratch=None) == _lib.STMP_OK
    assert fwd(K=4) == _lib.STMP_EUNSUPPORTED
    assert fwd(K=0) == _lib.STMP_EUNSUPPORTED
    assert fwd(out=65) == _lib.STMP_EUNSUPPORTED
    assert fwd(cin=65, out=64) == _lib.STMP_EUNSUPPORTED
    assert fwd(d=65) == _lib.STMP_EUNSUPPORTED
    assert fwd(n=4097) == _lib.STMP_EUNSUPPORTED
    assert fwd(x=ctypes.c_void_p(buf.data_ptr() + 2)) == _lib.STMP_ESHAPE
    assert L.stmp_agcrn_supported(2, 4096, 64, 64, 3, 64) == 1 and L.stmp_agcrn_supported(2, 10, 0, 4, 2, 5) == 0
    assert L.stmp_agcrn_supported(8388607, 1, 64, 64, 2, 5) == 1 and L.stmp_agcrn_supported(8388608, 1, 1, 1, 2, 5) == 0
    assert fwd(b=8388608) == _lib.STMP_EUNSUPPORTED                  # dT's 32-bit reduction length
    assert L.stmp_agcrn_scratch_bytes(2, 10, 3, 4, 4) == 0 and L.stmp_agcrn_workspace_bytes(-1, 10, 3, 4, 2) == 0
    assert L.stmp_agcrn_bwd(2, 10, 3, 4, 2, 5, p, p, None, p, p, p, p, p, None, p, p, *([None] * 7), st) == _lib.STMP_EINVAL
    torch.cuda.synchronize()
