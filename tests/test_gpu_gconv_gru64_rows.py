"""GConvGRU at 64 hidden channels on the 64-wide row-split cell kernels (`stmp_gru_wide_rows_*`, DESIGN §4n), which serve every graph
size at that width: the tutorial pattern against the unmodified reference (tests/golden/make_goldens_gconvgru64.py), fused and with
`fused_training = False`; every shape of the envelope against float64 with the criterion of test_gpu_rows_envelope.py (at most 4x the
fp32 op-for-op error plus 2^-20 of the tensor's scale) on graphs of 1 to 50 000 nodes; which kernels ran; bit-equality of the training and
inference forwards and of repeated backwards; loss-scale equivariance; launch counts; a captured WikiMaths step; routing; the C ABI's
errors."""
import ctypes
import itertools

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU
from pytorch_geometric_temporal_b200.plan import GraphPlan
from gconvgru64_seq import carried_h0, load, model_for, run_chickenpox, run_wikimaths
from gconvgru_seq import chickenpox_train_split
from test_gpu_rows_envelope import _check_err, _counted, _float64, _loss_grads, _or_zeros, _tensors, make_graph
from wikimaths_seq import load as load_wikimaths

pytestmark = pytest.mark.gpu
DEV = "cuda"
WIDE = ("k_gru_wide_rows_fwd_a", "k_gru_wide_rows_fwd_b", "k_gru_wide_rows_bwd_a", "k_gru_wide_rows_bwd_b", "k_gru_wide_rows_bwd_c",
        "k_gru_wide_rows_wgrad", "k_gru_wide_rows_wgrad_reduce")
NARROW = ("k_gru_rows_fwd_a", "k_gru_rows_fwd_b", "k_gru_rows_bwd_a", "k_gru_rows_bwd_b", "k_gru_rows_bwd_c", "k_gru_rows_wgrad_reduce",
          "k_gru_bwd_seq", "k_dcrnn_seq_tc", "k_dcrnn_wgrad")
WIKI = ["K2_sym", "K1_sym", "K2_rw", "K2_sym_carried"]


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _close_grad(got, want):
    _close(got, want, 1e-3, 1e-3 * want.abs().max().item() + 1e-6)


def _wide(c):
    return {k: v for k, v in c.items() if k in WIDE}


def _launches(given, want_dx, want_dh, K, train=True):
    """The 64-wide launches of one step."""
    w = {"k_gru_wide_rows_fwd_a": 1, "k_gru_wide_rows_fwd_b": int(given)}
    if train:
        w.update({"k_gru_wide_rows_bwd_a": 1, "k_gru_wide_rows_bwd_b": int(given), "k_gru_wide_rows_bwd_c": int(K == 2 and (want_dx or want_dh)),
                  "k_gru_wide_rows_wgrad": 1, "k_gru_wide_rows_wgrad_reduce": 1})
    return {k: v for k, v in w.items() if v}


# ---- 1. goldens from the unmodified reference ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wiki(golden_dir):
    g = load_wikimaths(golden_dir)
    return g["edge_index"].to(DEV), g["edge_weight"].to(DEV), g["X"].to(DEV), g["Y"].to(DEV)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", WIKI)
def test_wikimaths_vs_reference_golden(golden_dir, wiki, case, fused):
    c = load(golden_dir)["cases"][case]
    ei, ew, X, Y = wiki
    m = model_for(c, DEV, fused)
    H0 = carried_h0(X.size(1)).to(DEV).requires_grad_(True) if "gH0" in c else None
    lam = None if c["lambda_max"] is None else c["lambda_max"].to(DEV)
    with _counted() as cnt:
        out, losses = run_wikimaths(m, X, Y, ei, ew, lam, H0)
    S = X.size(0)
    if fused:
        want = {"k_gru_wide_rows_fwd_a": S, "k_gru_wide_rows_bwd_a": S, "k_gru_wide_rows_wgrad": S, "k_gru_wide_rows_wgrad_reduce": S}
        if H0 is not None:
            want.update({"k_gru_wide_rows_fwd_b": S, "k_gru_wide_rows_bwd_b": S, "k_gru_wide_rows_bwd_c": S})
        assert _wide(cnt) == want and "k_spmm" not in cnt, cnt
    else:
        assert _wide(cnt) == {}, cnt
    _close(out, c["out"])
    _close(losses, c["losses"])
    for k, p in m.named_parameters():
        _close_grad(p.grad, c["grads"][k])
    if H0 is not None:                  # dL/dH0 is ~1/N per entry and sums six steps: fp32 cancellation; test_carried_recurrence_vs_float64
        _close(H0.grad, c["gH0"], 1e-3, 4e-3 * c["gH0"].abs().max().item())   # holds it to the float64 criterion


@pytest.mark.parametrize("fused", [True, False])
def test_chickenpox_epoch_vs_reference_golden(golden_dir, fused):
    c = load(golden_dir)["cases"]["chickenpox"]
    ei, ew, X, Y = chickenpox_train_split()
    m = model_for(c, DEV, fused, node_features=4)
    with _counted() as cnt:
        out, cost = run_chickenpox(m, X.to(DEV), Y.to(DEV), ei.to(DEV), ew.to(DEV))
        cost.backward()
    S = X.size(0)
    if fused:
        assert _wide(cnt) == {"k_gru_wide_rows_fwd_a": S, "k_gru_wide_rows_bwd_a": S, "k_gru_wide_rows_wgrad": S,
                              "k_gru_wide_rows_wgrad_reduce": S}, cnt
    else:
        assert _wide(cnt) == {}, cnt
    assert not [k for k in cnt if k in NARROW], cnt
    _close(out, c["out"])
    _close(cost, c["cost"])
    for k, p in m.named_parameters():
        _close_grad(p.grad, c["grads"][k])


# ---- 2. the envelope against float64 ------------------------------------------------------------------------------------------------
def _model(cin, K, norm, bias, seed):
    torch.manual_seed(seed)
    m = GConvGRU(cin, 64, K, normalization=norm, bias=bias).to(DEV)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("bias"):
                p.copy_(torch.randn_like(p) * 0.1)
    return m


def _lam(norm):
    return torch.tensor(1.7, device=DEV) if norm == "rw" else None


def _hub_graph(N, seed, deg=6):
    """Random weighted directed graph with a hub of 1200 in-edges (node 0), one of 1200 out-edges (node 1) and 17 isolated nodes."""
    g = torch.Generator().manual_seed(seed)
    live = N - 17
    src = torch.randint(0, live, (deg * live,), generator=g)
    dst = torch.randint(0, live, (deg * live,), generator=g)
    src = torch.cat([src, torch.randperm(live, generator=g)[:1200], torch.ones(1200, dtype=torch.long)])
    dst = torch.cat([dst, torch.zeros(1200, dtype=torch.long), torch.randperm(live, generator=g)[:1200]])
    keep = src != dst
    ei = torch.unique(torch.stack([src[keep], dst[keep]]), dim=1)
    return ei.to(DEV), (torch.rand(ei.size(1), generator=g) + 0.1).to(DEV)


def _case(errs, m, ei, ew, n, norm, given, want_dx, want_dh, seed, what):
    """One step on the 64-wide kernels against float64: output and every wanted gradient; unwanted ones come back as None."""
    lam = _lam(norm)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(n, m.in_channels, device=DEV, generator=gen)
    H = 0.5 * torch.randn(n, 64, device=DEV, generator=gen)
    wgt = torch.randn(n, 64, device=DEV, generator=gen)
    want_dh = want_dh and given
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    x64, h64 = X.double().requires_grad_(True), H.double().requires_grad_(True)
    with _float64():
        o64 = R.gconv_gru_cell(p64, x64, ei, ew.double(), h64 if given else torch.zeros_like(h64), lambda_max=None if lam is None else lam.double(),
                               normalization=norm)
    g64 = _loss_grads([o64], [wgt.double()], [x64, h64] + [p64[k] for k in names])
    m.fused_training = False
    m.zero_grad(set_to_none=True)
    x32, h32 = X.clone().requires_grad_(True), H.clone().requires_grad_(True)
    o32 = m(x32, ei, ew, h32 if given else None, lambda_max=lam)
    g32 = _loss_grads([o32], [wgt], [x32, h32] + params)
    m.fused_training = True
    with torch.no_grad(), _counted() as c:
        inf = m(X, ei, ew, H if given else None, lambda_max=lam)
    assert _wide(c) == _launches(given, False, False, m.K, train=False), (what, c)
    m.zero_grad(set_to_none=True)
    xf, hf = X.clone().requires_grad_(want_dx), H.clone().requires_grad_(want_dh)
    with _counted() as c:
        of = m(xf, ei, ew, hf if given else None, lambda_max=lam)
        gf = _loss_grads([of], [wgt], [xf, hf] + params)
    assert _wide(c) == _launches(given, want_dx, want_dh, m.K), (what, c)
    assert "k_spmm" not in c and not [k for k in c if k in NARROW], (what, c)
    assert torch.equal(of.detach(), inf), (what, "training forward differs from inference")
    _check_err(errs, "gru_wide_rows", of, o32, o64, what + ("H'",))
    for label, want, got, r32, r64 in zip(["dX", "dH"] + names, [want_dx, want_dh] + [True] * len(names), gf, g32, g64):
        if not want:
            assert got is None, (what, label, "unwanted gradient")
            continue
        assert got is not None, (what, label)
        _check_err(errs, "gru_wide_rows", got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (label,))


CONFIGS = list(itertools.product((1, 4, 5, 14, 16), (1, 2)))           # (cin, K); K = 2 at cin = 16 fills the 160-column weight row
GEOMETRIES = [("ring", n) for n in (1, 2, 15, 16, 17, 33)] + [("mod4", 207), ("hubs", 208), ("random", 1068), ("hub_graph", 2600)]


def _graph(kind, n):
    if kind == "hub_graph":
        return _hub_graph(n, 5)
    return _tensors(make_graph(kind, n))


@pytest.mark.parametrize("kind,n", GEOMETRIES, ids=[f"{k}-N{n}" for k, n in GEOMETRIES])
def test_envelope_vs_float64(kind, n):
    """Every (cin, K) on every geometry; the normalization, the bias, H given or None and the X / H gradients cycle so each meets each."""
    ei, ew = _graph(kind, n)
    gi = GEOMETRIES.index((kind, n))
    errs = []
    for idx, (cin, K) in enumerate(CONFIGS):
        norm = ("sym", "rw")[(idx + gi) % 2]
        bias = bool((idx + gi // 2) % 2)
        given = bool((idx + gi) >> 1 & 1)
        m = _model(cin, K, norm, bias, seed=idx + n)
        _case(errs, m, ei, ew, n, norm, given, bool((idx + gi) >> 2 & 1) or idx % 3 == 0, True, 31 * n + idx, (kind, n, cin, K, norm, bias, given))
    assert not errs, errs[:6]


@pytest.mark.parametrize("K", [1, 2])
def test_state_and_gradient_flags_vs_float64(K):
    """H None or given, X / H gradients wanted or not, with and without bias, both normalizations."""
    n = 33
    ei, ew = _tensors(make_graph("mod4", n))
    errs = []
    for i, (given, want_dx, want_dh, bias, norm) in enumerate(itertools.product((False, True), (False, True), (False, True), (False, True),
                                                                                 ("sym", "rw"))):
        if want_dh and not given:
            continue
        m = _model(5, K, norm, bias, seed=K + i)
        _case(errs, m, ei, ew, n, norm, given, want_dx, want_dh, i, (K, given, want_dx, want_dh, bias, norm))
    assert not errs, errs[:6]


def test_a_50000_node_graph_vs_float64():
    n = 50000
    ei, ew = _hub_graph(n, 7)
    errs = []
    for given in (False, True):
        _case(errs, _model(14, 2, "sym", True, seed=3), ei, ew, n, "sym", given, True, True, 5, ("50000", given))
    assert not errs, errs[:6]


def test_carried_recurrence_vs_float64():
    """Five steps with H fed back and one backward through all of them."""
    n, cin, K, steps = 129, 14, 2, 5
    ei, ew = _tensors(make_graph("mod4_out", n))
    m = _model(cin, K, "sym", True, seed=11)
    gen = torch.Generator(device=DEV).manual_seed(2)
    X = torch.randn(steps, n, cin, device=DEV, generator=gen)
    H0 = 0.5 * torch.randn(n, 64, device=DEV, generator=gen)
    wgts = [torch.randn(n, 64, device=DEV, generator=gen) for _ in range(steps)]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]

    def run(dtype, step):
        x, h = X.to(dtype, copy=True).requires_grad_(True), H0.to(dtype, copy=True).requires_grad_(True)
        state, outs = h, []
        for t in range(steps):
            state = step(x[t], state)
            outs.append(state)
        return x, h, outs
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    with _float64():
        x64, h64, o64 = run(torch.float64, lambda x, h: R.gconv_gru_cell(p64, x, ei, ew.double(), h, lambda_max=None, normalization="sym"))
    g64 = _loss_grads(o64, [w.double() for w in wgts], [x64, h64] + [p64[k] for k in names])
    m.fused_training = False
    m.zero_grad(set_to_none=True)
    x32, h32, o32 = run(torch.float32, lambda x, h: m(x, ei, ew, h))
    g32 = _loss_grads(o32, wgts, [x32, h32] + params)
    m.fused_training = True
    m.zero_grad(set_to_none=True)
    with _counted() as c:
        xf, hf, of = run(torch.float32, lambda x, h: m(x, ei, ew, h))
        gf = _loss_grads(of, wgts, [xf, hf] + params)
    assert _wide(c) == {k: steps * v for k, v in _launches(True, True, True, K).items()}, c
    errs = []
    for label, got, r32, r64 in zip(["out", "dX", "dH0"] + names, [torch.stack(of)] + gf, [torch.stack(o32)] + g32, [torch.stack(o64)] + g64):
        _check_err(errs, "gru_wide_rows", got, r32, r64, ("recurrence", label))
    assert not errs, errs[:6]


# ---- 3. bit-exactness, loss scale, launch counts, CUDA graph ------------------------------------------------------------------------
def test_training_forward_is_bit_equal_to_inference_and_backward_is_deterministic(wiki):
    ei, ew, X, _ = wiki
    for K in (1, 2):
        m = _model(14, K, "sym", True, seed=K)
        H = 0.5 * torch.randn(X.size(1), 64, device=DEV)
        w = torch.randn(X.size(1), 64, device=DEV)
        for h in (H, None):
            out = m(X[1], ei, ew, h)
            with torch.no_grad():
                assert torch.equal(out.detach(), m(X[1], ei, ew, h))

            def grads():
                m.zero_grad(set_to_none=True)
                xl = X[1].clone().requires_grad_(True)
                hl = None if h is None else h.clone().requires_grad_(True)
                (m(xl, ei, ew, hl) * w).sum().backward()
                return [xl.grad] + ([hl.grad] if hl is not None else []) + [p.grad.clone() for p in m.parameters()]
            for a, b in zip(grads(), grads()):
                assert torch.equal(a, b)


@pytest.mark.parametrize("carried", [False, True])
def test_gradients_scale_with_a_power_of_two_loss_scale_bit_for_bit(golden_dir, wiki, carried):
    c = load(golden_dir)["cases"]["K2_sym_carried" if carried else "K2_sym"]
    ei, ew, X, Y = wiki

    def grads(scale):
        m = model_for(c, DEV, True)
        H0 = carried_h0(X.size(1)).to(DEV).requires_grad_(True) if carried else None
        h, total = H0, 0
        for t in range(X.size(0)):
            h = hh = m.recurrent(X[t], ei, ew, h)
            if not carried:
                h = None
            total = total + torch.mean((m.linear(torch.relu(hh)).squeeze() - Y[t]) ** 2)
        (total * scale).backward()
        return [p.grad for p in m.parameters()] + ([H0.grad] if carried else [])
    base = grads(1.0)
    for e in (-24, 8):
        for a, b in zip(grads(2.0 ** e), base):
            assert torch.equal(a, b * 2.0 ** e)


def test_launch_counts(wiki):
    ei, ew, X, _ = wiki
    m = _model(14, 2, "sym", True, seed=0)
    x = X[0]
    H = 0.5 * torch.randn(x.size(0), 64, device=DEV)
    w = torch.randn(x.size(0), 64, device=DEV)
    Hl = H.clone().requires_grad_(True)
    (m(x, ei, ew, Hl) * w).sum().backward()                    # warm: plan, packed weights, workspaces
    for h, want in ((H, 2), (None, 1)):
        n0 = _lib.launch_count()
        with torch.no_grad():
            m(x, ei, ew, h)
        assert _lib.launch_count() - n0 == want
    n0 = _lib.launch_count()
    out = m(x, ei, ew)                                         # the tutorial: H = None, X needs no gradient
    assert _lib.launch_count() - n0 == 1
    (out * w).sum().backward()
    assert _lib.launch_count() - n0 == 4                       # + bwd_a, wgrad contraction, reduce
    xl = x.clone().requires_grad_(True)
    n0 = _lib.launch_count()
    with _counted() as c:
        out = m(xl, ei, ew, Hl)
        assert _lib.launch_count() - n0 == 2
        (out * w).sum().backward()
    assert _lib.launch_count() - n0 == 7
    assert _wide(c) == {k: 1 for k in WIDE} and "k_spmm" not in c


def test_cuda_graph_replay_of_the_wikimaths_tutorial_step(golden_dir, wiki):
    """The tutorial step at 64 channels (H = None, MSE, backward, Adam(lr = 0.01)) captured once and replayed over the snapshots equals
    the same steps run eagerly."""
    c = load(golden_dir)["cases"]["K2_sym"]
    ei, ew, X, Y = wiki
    m = model_for(c, DEV, True)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    xs, ys = X[0].clone(), Y[0].clone()

    def step():
        cost = torch.mean((m.linear(torch.relu(m.recurrent(xs, ei, ew))).squeeze() - ys) ** 2)
        cost.backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
        return cost

    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step()
    m.load_state_dict(c["state"])
    for s in opt.state.values():
        for v in s.values():
            v.zero_()
    replay = []
    with _counted() as cnt:
        for t in range(X.size(0)):
            xs.copy_(X[t])
            ys.copy_(Y[t])
            graph.replay()
            replay.append(loss.detach().clone())
    torch.cuda.synchronize()
    assert _wide(cnt) == {}                                    # replays launch nothing through the library
    m_e = model_for(c, DEV, True)
    opt_e = torch.optim.Adam(m_e.parameters(), lr=0.01, capturable=True)      # the same update arithmetic as the captured step
    for t in range(X.size(0)):
        with _counted() as cnt:
            cost = torch.mean((m_e.linear(torch.relu(m_e.recurrent(X[t], ei, ew))).squeeze() - Y[t]) ** 2)
            cost.backward()
        assert cnt.get("k_gru_wide_rows_bwd_a") == 1
        opt_e.step()
        opt_e.zero_grad()
        _close(replay[t], cost.detach(), 1e-5, 1e-7)
    for p, pe in zip(m.parameters(), m_e.parameters()):
        _close(p, pe, 1e-5, 1e-6)


# ---- 4. routing and the C ABI ---------------------------------------------------------------------------------------------------------
def _ring(N):
    s = torch.arange(N, device=DEV)
    return torch.cat([torch.stack([s, (s + 1) % N]), torch.stack([(s + 1) % N, s])], dim=1)


def test_routing():
    """At 64, in_channels 17, K = 3 and 3-D X stay op-for-op; the 32-wide routes are unchanged (one-SM kernels on graphs that fit one SM,
    the 32-wide row-split kernels above)."""
    e300 = _ring(300)
    cases = [(GConvGRU(17, 64, 2), torch.randn(300, 17, device=DEV), torch.randn(300, 64, device=DEV)),
             (GConvGRU(4, 64, 3), torch.randn(300, 4, device=DEV), torch.randn(300, 64, device=DEV)),
             (GConvGRU(4, 64, 2), torch.randn(2, 300, 4, device=DEV), torch.randn(2, 300, 64, device=DEV))]
    for mod, x, h in cases:
        mod = mod.to(DEV)
        for grad in (False, True):
            with _counted() as c, torch.set_grad_enabled(grad):
                mod(x, e300, None, h)
            assert _wide(c) == {} and not [k for k in c if k in NARROW], c
    ei, ew, _, _ = chickenpox_train_split()
    ei, ew = ei.to(DEV), ew.to(DEV)
    for cin, kernel in ((4, "k_dcrnn_seq_tc"), (5, "k_spmm")):
        m = GConvGRU(cin, 32, 2).to(DEV)
        x, h = torch.randn(20, cin, device=DEV), torch.randn(20, 32, device=DEV).requires_grad_(True)
        with _counted() as c:
            with torch.no_grad():
                m(x, ei, ew, h)
            m(x, ei, ew, h).sum().backward()
        assert c.get(kernel, 0) > 0 and _wide(c) == {} and "k_gru_rows_fwd_a" not in c, c
    m = GConvGRU(4, 32, 2).to(DEV)
    with _counted() as c:
        m(torch.randn(208, 4, device=DEV), _ring(208), None, torch.randn(208, 32, device=DEV).requires_grad_(True)).sum().backward()
    assert c.get("k_gru_rows_bwd_a") == 1 and _wide(c) == {}, c
    m = GConvGRU(4, 64, 2).to(DEV)                              # 20 nodes at 64 channels: the 64-wide row-split kernels
    with _counted() as c:
        m(torch.randn(20, 4, device=DEV), ei, ew, torch.randn(20, 64, device=DEV).requires_grad_(True)).sum().backward()
    assert c.get("k_gru_wide_rows_bwd_a") == 1 and not [k for k in c if k in NARROW], c


def test_abi_errors():
    ei, ew, _, _ = chickenpox_train_split()
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 20, "sym")
    L = _lib.lib()
    h = cheb.handle
    buf = torch.zeros(1 << 20, device=DEV)
    p, q = _lib.ptr(buf), ctypes.c_void_p(buf.data_ptr() + 4)       # q: 4-byte aligned only
    r = ctypes.c_void_p(buf.data_ptr() + 2)                         # r: misaligned
    assert L.stmp_gru_rows_supported(h, 1, 16, 64) == 1 and L.stmp_gru_rows_supported(h, 0, 1, 64) == 1
    assert L.stmp_gru_rows_supported(h, 1, 17, 64) == 0 and L.stmp_gru_rows_supported(h, 2, 4, 64) == 0
    assert L.stmp_gru_rows_supported(h, 1, 4, 48) == 0 and L.stmp_gru_rows_supported(None, 1, 4, 64) == 0
    ld = ops.gru_rows_basis_ld(1, 4, 64)
    assert ld == 136
    fwd = lambda n_ops, cin, x=p, hh=p, S1=p, ldv=ld: L.stmp_gru_wide_rows_fwd(h, n_ops, cin, x, hh, p, p, p, p, p, S1, p, ldv, None)
    assert fwd(1, 17) == _lib.STMP_EUNSUPPORTED and fwd(2, 4) == _lib.STMP_EUNSUPPORTED
    assert fwd(1, 4, x=None) == _lib.STMP_EINVAL
    assert fwd(1, 4, ldv=ops.gru_rows_basis_ld(1, 4)) == _lib.STMP_ESHAPE and fwd(1, 4, x=r) == _lib.STMP_ESHAPE
    assert fwd(1, 4, S1=q) == _lib.STMP_ESHAPE
    assert L.stmp_gru_wide_rows_fwd(h, 1, 4, p, None, p, p, None, p, p, p, p, ld, None) == _lib.STMP_EINVAL      # S2 without h
    assert L.stmp_gru_wide_rows_fwd(None, 1, 4, p, p, p, p, p, p, p, p, p, ld, None) == _lib.STMP_EINVAL
    bwd = lambda cin, g=p, hh=p, dh=p: L.stmp_gru_wide_rows_bwd(h, 1, cin, g, hh, p, p, p, p, p, p, dh, None)
    assert bwd(17) == _lib.STMP_EUNSUPPORTED and bwd(4, g=None) == _lib.STMP_EINVAL and bwd(4, hh=None) == _lib.STMP_EINVAL
    assert bwd(4, g=r) == _lib.STMP_ESHAPE
    wg = lambda n_ops, ldv, S1=p: L.stmp_gru_wide_rows_wgrad(n_ops, 4, 20, ldv, S1, p, p, p, p, p, p, None)
    assert wg(1, ld + 8) == _lib.STMP_ESHAPE and wg(2, ld) == _lib.STMP_EUNSUPPORTED and wg(1, ld, S1=None) == _lib.STMP_EINVAL
    assert wg(1, ld, S1=q) == _lib.STMP_ESHAPE
    assert L.stmp_gru_wide_rows_pack_weights(1, 17, p, p, None, None, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_gru_wide_rows_pack_weights(1, 4, None, p, None, None, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_gru_wide_rows_pack_weights(1, 4, p, p, p, None, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_gru_wide_rows_wgrad_workspace_bytes(1, 16) > 0 and L.stmp_gru_wide_rows_scratch_bytes(h) == 20 * 320 * 4
    assert L.stmp_gru_wide_rows_scratch_bytes(None) == 0
