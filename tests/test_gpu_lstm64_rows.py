"""GConvLSTM and GCLSTM at 64 hidden channels on the 64-wide row-split LSTM cell kernels (`stmp_lstm_wide_rows_*`, DESIGN §4o): the
tutorial patterns against the float64 oracle, itself held to the unmodified reference (tests/golden/make_goldens_lstm64.py), fused and with
`fused_training = False`; every
shape of the envelope against float64 with the criterion of test_gpu_rows_envelope.py (at most 4x the fp32 op-for-op error plus 2^-20 of
the tensor's scale) on graphs of 1 to 50 000 nodes; which kernels ran; bit-equality of the training and inference forwards and of repeated
backwards; loss-scale equivariance; the weight-gradient reduce recomputed bit for bit; launch counts; a captured WikiMaths step; routing;
the C ABI's errors."""
import ctypes
import itertools

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib, ops
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvLSTM
from pytorch_geometric_temporal_b200.plan import GraphPlan
from gconvgru_seq import chickenpox_train_split
from lstm64_seq import carried_state, check_reference, load, model_for, oracle_run, run, seeded_state
from test_gpu_rows_envelope import _check_err, _counted, _float64, _loss_grads, _or_zeros, _tensors, make_graph
from test_gpu_wgrad_reduce import _ar, _check, _equal, _operands, _parts, _randn, _rows, _sms, _sum, _workspace, PARTS, NAN
from wikimaths_seq import load as load_wikimaths

pytestmark = pytest.mark.gpu
DEV = "cuda"
WIDE = ("k_lstm_wide_rows_fwd", "k_lstm_wide_rows_bwd_a", "k_lstm_wide_rows_bwd_b", "k_lstm_wide_rows_wgrad", "k_lstm_wide_rows_wgrad_reduce")
NARROW = ("k_lstm_rows_fwd", "k_lstm_rows_bwd_a", "k_lstm_rows_bwd_b", "k_lstm_rows_wgrad_reduce", "k_dcrnn_wgrad", "k_lstm_gate_bwd")
MODULES = {"gconv_lstm": GConvLSTM, "gc_lstm": GCLSTM}
ORACLE = {"gconv_lstm": R.gconv_lstm_cell, "gc_lstm": R.gc_lstm_cell}
WIKI = ["K2_sym", "K1_sym", "K2_rw", "K2_sym_carried"]


def _close(got, want, rtol=1e-4, atol=1e-5):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=rtol, atol=atol), f"max abs err {(got - want).abs().max():.3e}"


def _close_grad(got, want):
    _close(got, want, 1e-3, 1e-3 * want.abs().max().item() + 1e-6)


def _wide(c):
    return {k: v for k, v in c.items() if k in WIDE}


def _rows_inference(cin, n):
    """Whether a no_grad call takes the 64-wide cell: the SpMM + wgmma route keeps in_channels % 4 == 0 on large graphs."""
    return cin % 4 != 0 or n < ops.LSTM_WIDE_ROWS_GEMM_NODES


def _launches(name, K, gather, train=True):
    """The 64-wide launches of one step; `gather`: dH (or, for GConvLSTM, dX) is wanted."""
    w = {"k_lstm_wide_rows_fwd": 1}
    if train:
        w.update({"k_lstm_wide_rows_bwd_a": 1, "k_lstm_wide_rows_bwd_b": int(K == 2 and gather), "k_lstm_wide_rows_wgrad": 1,
                  "k_lstm_wide_rows_wgrad_reduce": 1})
    return {k: v for k, v in w.items() if v}


# ---- 1. goldens from the unmodified reference ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wiki(golden_dir):
    g = load_wikimaths(golden_dir)
    return g["edge_index"].to(DEV), g["edge_weight"].to(DEV), g["X"].to(DEV), g["Y"].to(DEV)


def _golden(c, fused, ei, ew, X, Y):
    """Case c on the module (fused or op for op) against the float64 oracle, element by element, once the oracle has matched the unmodified
    reference's fingerprints and cost."""
    m = model_for(c, DEV, fused)
    n = X.size(1)
    carried = "gH0" in c["fingerprints"]
    H0 = carried_state(n, 7, 13, 17).to(DEV).requires_grad_(True) if carried else None
    C0 = carried_state(n, 5, 11, 19).to(DEV).requires_grad_(True) if carried else None
    lam = None if c["lambda_max"] is None else c["lambda_max"].to(DEV)
    H064 = None if H0 is None else H0.detach().double().requires_grad_(True)
    C064 = None if C0 is None else C0.detach().double().requires_grad_(True)
    out64, cost64, leaves = oracle_run(c, X, Y, ei, ew, lam, H064, C064)
    cost64.backward()
    check_reference(c, out64, cost64, {k: v.grad for k, v in leaves.items()}, *((H064.grad, C064.grad) if carried else ()))
    with _counted() as cnt:
        out, cost = run(m, X, Y, ei, ew, lam, H0, C0)
        cost.backward()
    S = X.size(0)
    if fused:                          # H and C are carried: only a step from H = None has no dH (and GCLSTM no dX to gather either)
        want = {"k_lstm_wide_rows_fwd": S, "k_lstm_wide_rows_bwd_a": S, "k_lstm_wide_rows_wgrad": S, "k_lstm_wide_rows_wgrad_reduce": S,
                "k_lstm_wide_rows_bwd_b": (S - (not carried)) if c["K"] == 2 else 0}
        assert _wide(cnt) == {k: v for k, v in want.items() if v} and "k_spmm" not in cnt, cnt
    else:
        assert _wide(cnt) == {}, cnt
    assert not [k for k in cnt if k in NARROW], cnt
    _close(out, out64)
    _close(cost, cost64)
    for k, p in m.named_parameters():
        _close_grad(p.grad, leaves[k].grad)
    if carried:                        # dL/dH0 and dL/dC0 sum every step: fp32 cancellation; test_carried_recurrence_vs_float64 holds them
        _close(H0.grad, H064.grad, 1e-3, 4e-3 * H064.grad.abs().max().item())   # to the float64 criterion
        _close(C0.grad, C064.grad, 1e-3, 4e-3 * C064.grad.abs().max().item())


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", WIKI)
@pytest.mark.parametrize("name", list(MODULES))
def test_wikimaths_vs_reference_golden(golden_dir, wiki, name, case, fused):
    c = load(golden_dir)["cases"][f"{name}/{case}"]
    ei, ew, X, Y = wiki
    _golden(c, fused, ei, ew, X, Y)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", list(MODULES))
def test_chickenpox_epoch_vs_reference_golden(golden_dir, name, fused):
    c = load(golden_dir)["cases"][f"{name}/chickenpox"]
    ei, ew, X, Y = chickenpox_train_split()
    _golden(c, fused, ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV))


# ---- 2. the envelope against float64 ------------------------------------------------------------------------------------------------
def _model(name, cin, K, norm, bias, seed):
    torch.manual_seed(seed)
    m = MODULES[name](cin, 64, K, normalization=norm, bias=bias).to(DEV)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("bias") or k.startswith("b_"):
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


def _case(errs, name, m, ei, ew, n, norm, given, want_dx, want_ds, seed, what):
    """One step on the 64-wide kernels against float64: H', C' and every wanted gradient; unwanted ones come back as None.  `given`: H and
    C given (else None); `want_ds`: their gradients wanted."""
    lam = _lam(norm)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    X = torch.randn(n, m.in_channels, device=DEV, generator=gen)
    H = 0.5 * torch.randn(n, 64, device=DEV, generator=gen)
    C = 0.5 * torch.randn(n, 64, device=DEV, generator=gen)
    wgts = [torch.randn(n, 64, device=DEV, generator=gen) for _ in range(2)]
    want_ds = want_ds and given
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    x64, h64, c64 = (t.double().requires_grad_(True) for t in (X, H, C))
    with _float64():
        o64 = ORACLE[name](p64, x64, ei, ew.double(), h64 if given else torch.zeros_like(h64), c64 if given else torch.zeros_like(c64),
                           lambda_max=None if lam is None else lam.double(), normalization=norm)
    g64 = _loss_grads(list(o64), [w.double() for w in wgts], [x64, h64, c64] + [p64[k] for k in names])
    m.fused_training = False
    m.zero_grad(set_to_none=True)
    x32, h32, c32 = (t.clone().requires_grad_(True) for t in (X, H, C))
    o32 = m(x32, ei, ew, h32 if given else None, c32 if given else None, lambda_max=lam)
    g32 = _loss_grads(list(o32), wgts, [x32, h32, c32] + params)
    m.fused_training = True
    with torch.no_grad(), _counted() as c:
        inf = m(X, ei, ew, H if given else None, C if given else None, lambda_max=lam)
    rows_inf = _rows_inference(m.in_channels, n)
    assert _wide(c) == (_launches(name, m.K, False, train=False) if rows_inf else {}), (what, c)
    m.zero_grad(set_to_none=True)
    xf, hf, cf = X.clone().requires_grad_(want_dx), H.clone().requires_grad_(want_ds), C.clone().requires_grad_(want_ds)
    with _counted() as c:
        of = m(xf, ei, ew, hf if given else None, cf if given else None, lambda_max=lam)
        gf = _loss_grads(list(of), wgts, [xf, hf, cf] + params)
    gather = want_ds or (name == "gconv_lstm" and want_dx)
    assert _wide(c) == _launches(name, m.K, gather), (what, c)
    assert "k_spmm" not in c and not [k for k in c if k in NARROW], (what, c)
    if rows_inf:
        assert torch.equal(of[0].detach(), inf[0]) and torch.equal(of[1].detach(), inf[1]), (what, "training forward differs from inference")
    for i in range(2):
        _check_err(errs, "lstm_wide_rows", of[i], o32[i], o64[i], what + (("H'", "C'")[i],))
    for label, want, got, r32, r64 in zip(["dX", "dH", "dC"] + names, [want_dx, want_ds, want_ds] + [True] * len(names), gf, g32, g64):
        if not want:
            assert got is None, (what, label, "unwanted gradient")
            continue
        assert got is not None, (what, label)
        _check_err(errs, "lstm_wide_rows", got, _or_zeros(r32, got), _or_zeros(r64, got.double()), what + (label,))


CONFIGS = list(itertools.product(MODULES, (1, 4, 5, 14, 16), (1, 2)))   # (module, cin, K); GConvLSTM K = 2 at cin 16: the 160-column row
GEOMETRIES = [("ring", n) for n in (1, 2, 15, 16, 17, 33)] + [("mod4", 207), ("hubs", 208), ("random", 1068), ("hub_graph", 2600)]


def _graph(kind, n):
    if kind == "hub_graph":
        return _hub_graph(n, 5)
    return _tensors(make_graph(kind, n))


@pytest.mark.parametrize("kind,n", GEOMETRIES, ids=[f"{k}-N{n}" for k, n in GEOMETRIES])
def test_envelope_vs_float64(kind, n):
    """Every (module, cin, K) on every geometry; the normalization, the bias, H / C given or None and the X / state gradients cycle so
    each meets each."""
    ei, ew = _graph(kind, n)
    gi = GEOMETRIES.index((kind, n))
    errs = []
    for idx, (name, cin, K) in enumerate(CONFIGS):
        norm = ("sym", "rw")[(idx + gi) % 2]
        bias = bool((idx + gi // 2) % 2)
        given = bool((idx + gi) >> 1 & 1)
        m = _model(name, cin, K, norm, bias, seed=idx + n)
        _case(errs, name, m, ei, ew, n, norm, given, bool((idx + gi) >> 2 & 1) or idx % 3 == 0, True, 31 * n + idx,
              (kind, n, name, cin, K, norm, bias, given))
    assert not errs, errs[:6]


@pytest.mark.parametrize("name", list(MODULES))
@pytest.mark.parametrize("K", [1, 2])
def test_state_and_gradient_flags_vs_float64(name, K):
    """H / C None or given, X / state gradients wanted or not, with and without bias, both normalizations."""
    n = 33
    ei, ew = _tensors(make_graph("mod4", n))
    errs = []
    for i, (given, want_dx, want_ds, bias, norm) in enumerate(itertools.product((False, True), (False, True), (False, True), (False, True),
                                                                                 ("sym", "rw"))):
        if want_ds and not given:
            continue
        m = _model(name, 5, K, norm, bias, seed=K + i)
        _case(errs, name, m, ei, ew, n, norm, given, want_dx, want_ds, i, (name, K, given, want_dx, want_ds, bias, norm))
    assert not errs, errs[:6]


def test_a_50000_node_graph_vs_float64():
    n = 50000
    ei, ew = _hub_graph(n, 7)
    errs = []
    for name in MODULES:
        for given in (False, True):
            _case(errs, name, _model(name, 14, 2, "sym", True, seed=3), ei, ew, n, "sym", given, True, True, 5, (name, "50000", given))
        _case(errs, name, _model(name, 16, 2, "sym", True, seed=4), ei, ew, n, "sym", True, True, True, 6, (name, "50000", 16))
    assert not errs, errs[:6]


@pytest.mark.parametrize("name", list(MODULES))
def test_carried_recurrence_vs_float64(name):
    """Five steps with H and C fed back and one backward through all of them."""
    n, cin, K, steps = 129, 14, 2, 5
    ei, ew = _tensors(make_graph("mod4_out", n))
    m = _model(name, cin, K, "sym", True, seed=11)
    gen = torch.Generator(device=DEV).manual_seed(2)
    X = torch.randn(steps, n, cin, device=DEV, generator=gen)
    H0 = 0.5 * torch.randn(n, 64, device=DEV, generator=gen)
    C0 = 0.5 * torch.randn(n, 64, device=DEV, generator=gen)
    wgts = [torch.randn(n, 64, device=DEV, generator=gen) for _ in range(2 * steps)]
    names = [k for k, _ in m.named_parameters()]
    params = [p for _, p in m.named_parameters()]

    def run(dtype, step):
        x, h, c = (t.to(dtype, copy=True).requires_grad_(True) for t in (X, H0, C0))
        state, outs = (h, c), []
        for t in range(steps):
            state = step(x[t], state)
            outs += list(state)
        return x, h, c, outs
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in m.state_dict().items()}
    with _float64():
        x64, h64, c64, o64 = run(torch.float64, lambda x, s: ORACLE[name](p64, x, ei, ew.double(), *s, lambda_max=None, normalization="sym"))
    g64 = _loss_grads(o64, [w.double() for w in wgts], [x64, h64, c64] + [p64[k] for k in names])
    m.fused_training = False
    m.zero_grad(set_to_none=True)
    x32, h32, c32, o32 = run(torch.float32, lambda x, s: m(x, ei, ew, *s))
    g32 = _loss_grads(o32, wgts, [x32, h32, c32] + params)
    m.fused_training = True
    m.zero_grad(set_to_none=True)
    with _counted() as c:
        xf, hf, cf, of = run(torch.float32, lambda x, s: m(x, ei, ew, *s))
        gf = _loss_grads(of, wgts, [xf, hf, cf] + params)
    assert _wide(c) == {k: steps * v for k, v in _launches(name, K, True).items()}, c
    errs = []
    for label, got, r32, r64 in zip(["out", "dX", "dH0", "dC0"] + names, [torch.stack(of)] + gf, [torch.stack(o32)] + g32,
                                    [torch.stack(o64)] + g64):
        _check_err(errs, "lstm_wide_rows", got, r32, r64, (name, "recurrence", label))
    assert not errs, errs[:6]


# ---- 3. bit-exactness, loss scale, the reduce, launch counts, CUDA graph ------------------------------------------------------------
@pytest.mark.parametrize("name", list(MODULES))
def test_training_forward_is_bit_equal_to_inference_and_backward_is_deterministic(wiki, name):
    """At cin = 14 every graph size takes the 64-wide cell for inference too (cin % 4 != 0)."""
    ei, ew, X, _ = wiki
    for K in (1, 2):
        m = _model(name, 14, K, "sym", True, seed=K)
        H = 0.5 * torch.randn(X.size(1), 64, device=DEV)
        C = 0.5 * torch.randn(X.size(1), 64, device=DEV)
        w = torch.randn(X.size(1), 64, device=DEV)
        for h, c in ((H, C), (None, None), (H, None)):
            out = m(X[1], ei, ew, h, c)
            with torch.no_grad(), _counted() as cnt:
                inf = m(X[1], ei, ew, h, c)
            assert cnt.get("k_lstm_wide_rows_fwd") == 1
            assert torch.equal(out[0].detach(), inf[0]) and torch.equal(out[1].detach(), inf[1])

            def grads():
                m.zero_grad(set_to_none=True)
                xl = X[1].clone().requires_grad_(True)
                hl = None if h is None else h.clone().requires_grad_(True)
                cl = None if c is None else c.clone().requires_grad_(True)
                a, b = m(xl, ei, ew, hl, cl)
                ((a + b) * w).sum().backward()
                return [xl.grad] + [t.grad for t in (hl, cl) if t is not None] + [p.grad.clone() for p in m.parameters()]
            for a, b in zip(grads(), grads()):
                assert torch.equal(a, b)


@pytest.mark.parametrize("name", list(MODULES))
def test_gradients_scale_with_a_power_of_two_loss_scale_bit_for_bit(wiki, name):
    ei, ew, X, Y = wiki
    n = X.size(1)

    def grads(scale):
        m = _model(name, 14, 2, "sym", True, seed=9)
        lin = torch.nn.Linear(64, 1).to(DEV)
        torch.manual_seed(1)
        torch.nn.init.normal_(lin.weight)
        H0 = carried_state(n, 7, 13, 17).to(DEV).requires_grad_(True)
        C0 = carried_state(n, 5, 11, 19).to(DEV).requires_grad_(True)
        h, c, total = H0, C0, 0
        for t in range(3):
            h, c = m(X[t], ei, ew, h, c)
            total = total + torch.mean((lin(torch.relu(h)).squeeze() - Y[t]) ** 2)
        (total * scale).backward()
        return [p.grad for p in m.parameters()] + [H0.grad, C0.grad]
    base = grads(1.0)
    for e in (-24, 8):
        for a, b in zip(grads(2.0 ** e), base):
            assert torch.equal(a, b * 2.0 ** e)


@pytest.mark.parametrize("peep", [True, False])
@pytest.mark.parametrize("parts", PARTS)
@pytest.mark.parametrize("variant", [_lib.LSTM_GCONV, _lib.LSTM_GC])
def test_wide_wgrad_reduce_is_the_fixed_order_sum(variant, parts, peep):
    """stmp_lstm_wide_rows_wgrad: k_wide_rows_wgrad<4> (one partial per (gate, CTA) of 32-row tiles), then k_wide_rows_wgrad_reduce<4>
    into dw [256][nb], db [256] and, from the per-CTA peephole sums k_lstm_rows_bwd_a<2> leaves in the scratch behind its N·80 floats,
    dpeep [192]; every element recomputed in float32 in the reduce's association (test_gpu_wgrad_reduce.py)."""
    torch.manual_seed(6 + variant)
    n_ops, cin = 1, 5
    nb, ld = ops.lstm_rows_nb(variant, n_ops, cin, 64), ops.lstm_rows_basis_ld(variant, n_ops, cin, 64)
    cap = 2 * _sms()
    rows = _rows(parts, 32, cap)
    n = _parts(rows, 32, cap)
    npp = _parts(rows, 16, cap)                                        # rows_grid(rows): the backward's CTAs
    S, = _operands(rows, ld)
    dpre = _randn(2, max(rows, 1), 128)
    scratch = _randn(rows * 80 + max(npp, 1) * 192)
    ws = _workspace(_lib.lib().stmp_lstm_wide_rows_wgrad_workspace_bytes(variant, n_ops, cin))
    dw = torch.full((256, nb), NAN, device=DEV)
    db = torch.full((256,), NAN, device=DEV)
    dpeep = torch.full((192,), NAN, device=DEV)
    _check(_lib.lib().stmp_lstm_wide_rows_wgrad(variant, n_ops, cin, rows, ld, _lib.ptr(S), _lib.ptr(dpre), _lib.ptr(scratch), _lib.ptr(ws),
                                                _lib.ptr(dw), _lib.ptr(db), _lib.ptr(dpeep) if peep else None, _lib.stream_ptr()))
    if rows == 0:
        assert not dw.any() and not db.any() and (not dpeep.any() if peep else torch.isnan(dpeep).all())
        return
    stride = ld * 64 + 64
    P = ws[:4 * n * stride].view(4, n, stride).cpu()
    row, m = torch.meshgrid(_ar(64), _ar(nb), indexing="ij")
    _equal(dw, torch.cat([_sum(P[g], m * 64 + row) for g in range(4)]))
    _equal(db, torch.cat([_sum(P[g], ld * 64 + _ar(64)) for g in range(4)]))
    if peep:
        _equal(dpeep, _sum(scratch[rows * 80:rows * 80 + npp * 192].view(npp, 192).cpu(), _ar(192)))
    else:
        assert torch.isnan(dpeep).all()


@pytest.mark.parametrize("name", list(MODULES))
def test_launch_counts(wiki, name):
    ei, ew, X, _ = wiki
    m = _model(name, 14, 2, "sym", True, seed=0)
    x = X[0]
    H = 0.5 * torch.randn(x.size(0), 64, device=DEV)
    w = torch.randn(x.size(0), 64, device=DEV)
    Hl, Cl = H.clone().requires_grad_(True), H.clone().requires_grad_(True)
    (m(x, ei, ew, Hl, Cl)[0] * w).sum().backward()             # warm: plan, packed weights, workspaces
    for h in (H, None):
        n0 = _lib.launch_count()
        with torch.no_grad():
            m(x, ei, ew, h, h)
        assert _lib.launch_count() - n0 == 1
    n0 = _lib.launch_count()
    out = m(x, ei, ew)                                         # the tutorial: H = C = None, X needs no gradient
    assert _lib.launch_count() - n0 == 1
    (out[0] * w).sum().backward()
    assert _lib.launch_count() - n0 == 4                       # + bwd_a, wgrad contraction, reduce
    xl = x.clone().requires_grad_(True)
    n0 = _lib.launch_count()
    with _counted() as c:
        out = m(xl, ei, ew, Hl, Cl)
        assert _lib.launch_count() - n0 == 1
        ((out[0] + out[1]) * w).sum().backward()
    assert _lib.launch_count() - n0 == 5
    assert _wide(c) == {k: 1 for k in WIDE} and "k_spmm" not in c


@pytest.mark.parametrize("name", list(MODULES))
def test_cuda_graph_replay_of_the_wikimaths_tutorial_step(golden_dir, wiki, name):
    """The tutorial step at 64 channels (H = C = None, MSE, backward, Adam(lr = 0.01)) captured once and replayed over the snapshots
    equals the same steps run eagerly."""
    c = load(golden_dir)["cases"][f"{name}/K2_sym"]
    ei, ew, X, Y = wiki
    m = model_for(c, DEV, True)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    xs, ys = X[0].clone(), Y[0].clone()

    def step():
        cost = torch.mean((m.linear(torch.relu(m.recurrent(xs, ei, ew)[0])).squeeze() - ys) ** 2)
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
    m.load_state_dict(seeded_state(c["module"], c["F"], c["K"], c["seed"]))
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
    opt_e = torch.optim.Adam(m_e.parameters(), lr=0.01, capturable=True)
    for t in range(X.size(0)):
        with _counted() as cnt:
            cost = torch.mean((m_e.linear(torch.relu(m_e.recurrent(X[t], ei, ew)[0])).squeeze() - Y[t]) ** 2)
            cost.backward()
        assert cnt.get("k_lstm_wide_rows_bwd_a") == 1
        opt_e.step()
        opt_e.zero_grad()
        _close(replay[t], cost.detach(), 1e-5, 1e-7)
    for p, pe in zip(m.parameters(), m_e.parameters()):
        _close(p, pe, 1e-5, 1e-6)


# ---- 4. routing and the C ABI ---------------------------------------------------------------------------------------------------------
def _ring(N):
    s = torch.arange(N, device=DEV)
    return torch.cat([torch.stack([s, (s + 1) % N]), torch.stack([(s + 1) % N, s])], dim=1)


@pytest.mark.parametrize("name", list(MODULES))
def test_routing(name):
    """At 64, in_channels 17, K = 3 and 3-D X stay off the row-split kernels; `no_grad` with in_channels % 4 == 0 takes the 64-wide cell
    below ops.LSTM_WIDE_ROWS_GEMM_NODES nodes and the SpMM + wgmma route from there on; fused_training = False trains op for op."""
    cls = MODULES[name]
    e300 = _ring(300)
    for mod, x in ((cls(17, 64, 2), torch.randn(300, 17, device=DEV)), (cls(4, 64, 3), torch.randn(300, 4, device=DEV)),
                   (cls(4, 64, 2), torch.randn(2, 300, 4, device=DEV))):
        mod = mod.to(DEV)
        h = torch.randn(*x.shape[:-1], 64, device=DEV)
        for grad in (False, True):
            with _counted() as c, torch.set_grad_enabled(grad):
                mod(x, e300, None, h, h)
            assert _wide(c) == {} and not [k for k in c if k in NARROW[:4]], c
    big = ops.LSTM_WIDE_ROWS_GEMM_NODES
    for n, cin, want in ((big - 1, 4, 1), (big, 4, 0), (big, 5, 1), (big, 16, 0)):
        mod = cls(cin, 64, 2).to(DEV)
        with torch.no_grad(), _counted() as c:
            mod(torch.randn(n, cin, device=DEV), _ring(n))
        assert c.get("k_lstm_wide_rows_fwd", 0) == want, (n, cin, c)
    mod = cls(4, 64, 2).to(DEV)
    mod.fused_training = False
    with _counted() as c:
        mod(torch.randn(300, 4, device=DEV), e300)[0].sum().backward()
    assert _wide(c) == {} and "k_spmm" in c, c
    mod.fused_training = True
    with _counted() as c:
        mod(torch.randn(300, 4, device=DEV), e300)[0].sum().backward()
    assert c.get("k_lstm_wide_rows_bwd_a") == 1 and not [k for k in c if k in NARROW], c


def test_abi_errors():
    ei, ew, _, _ = chickenpox_train_split()
    cheb = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 20, "sym")
    L = _lib.lib()
    h = cheb.handle
    GCV, GC = _lib.LSTM_GCONV, _lib.LSTM_GC
    buf = torch.zeros(1 << 20, device=DEV)
    p, q = _lib.ptr(buf), ctypes.c_void_p(buf.data_ptr() + 4)       # q: 4-byte aligned only
    r = ctypes.c_void_p(buf.data_ptr() + 2)                         # r: misaligned
    for v in (GCV, GC):
        assert L.stmp_lstm_rows_supported(h, v, 1, 16, 64) == 1 and L.stmp_lstm_rows_supported(h, v, 0, 1, 64) == 1
        assert L.stmp_lstm_rows_supported(h, v, 1, 17, 64) == 0 and L.stmp_lstm_rows_supported(h, v, 2, 4, 64) == 0
        assert L.stmp_lstm_rows_supported(h, v, 1, 4, 48) == 0 and L.stmp_lstm_rows_supported(None, v, 1, 4, 64) == 0
    assert ops.lstm_rows_basis_ld(GCV, 1, 4, 64) == 136 and ops.lstm_rows_basis_ld(GC, 1, 4, 64) == 136
    assert ops.lstm_rows_nb(GC, 1, 5, 64) == 133 and ops.lstm_rows_basis_ld(GC, 1, 5, 64) == 136
    ld = ops.lstm_rows_basis_ld(GCV, 1, 4, 64)
    fwd = lambda n_ops, cin, v=GCV, x=p, S=p, ldv=ld: L.stmp_lstm_wide_rows_fwd(h, v, n_ops, cin, x, p, p, p, p, p, p, p, p, S, ldv, None)
    assert fwd(1, 17) == _lib.STMP_EUNSUPPORTED and fwd(2, 4) == _lib.STMP_EUNSUPPORTED and fwd(1, 4, v=2) == _lib.STMP_EINVAL
    assert fwd(1, 4, x=None) == _lib.STMP_EINVAL
    assert fwd(1, 4, ldv=ops.lstm_rows_basis_ld(GCV, 1, 4)) == _lib.STMP_ESHAPE and fwd(1, 4, x=r) == _lib.STMP_ESHAPE
    assert fwd(1, 4, S=q) == _lib.STMP_ESHAPE
    assert L.stmp_lstm_wide_rows_fwd(None, GCV, 1, 4, p, p, p, p, p, p, p, p, p, p, ld, None) == _lib.STMP_EINVAL
    bwd = lambda cin, cn=p, c=p, dc=p, dpre=p: L.stmp_lstm_wide_rows_bwd(h, GCV, 1, cin, p, p, c, cn, p, p, p, p, dpre, p, p, dc, None)
    assert bwd(17) == _lib.STMP_EUNSUPPORTED and bwd(4, cn=None) == _lib.STMP_EINVAL and bwd(4, c=None) == _lib.STMP_EINVAL
    assert bwd(4, dpre=q) == _lib.STMP_ESHAPE
    wg = lambda n_ops, ldv, S=p, scratch=p: L.stmp_lstm_wide_rows_wgrad(GCV, n_ops, 4, 20, ldv, S, p, scratch, p, p, p, p, None)
    assert wg(1, ld + 8) == _lib.STMP_ESHAPE and wg(2, ld) == _lib.STMP_EUNSUPPORTED and wg(1, ld, S=None) == _lib.STMP_EINVAL
    assert wg(1, ld, S=q) == _lib.STMP_ESHAPE and wg(1, ld, scratch=None) == _lib.STMP_EINVAL     # dpeep reads the scratch
    assert L.stmp_lstm_wide_rows_pack_weights(GCV, 1, 17, p, p, None, None, p, p, p, None) == _lib.STMP_EUNSUPPORTED
    assert L.stmp_lstm_wide_rows_pack_weights(GCV, 1, 4, None, p, None, None, p, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_lstm_wide_rows_pack_weights(GCV, 1, 4, p, p, p, None, p, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_lstm_wide_rows_pack_weights(GC, 1, 4, p, p, p, p, p, p, p, None) == _lib.STMP_EINVAL
    assert L.stmp_lstm_wide_rows_wgrad_workspace_bytes(GCV, 1, 16) > 0 and L.stmp_lstm_wide_rows_wgrad_workspace_bytes(GCV, 1, 17) == 0
    assert L.stmp_lstm_wide_rows_scratch_bytes(h) == (20 * 80 + 2 * 192) * 4           # 20 rows: two 16-row tiles of peephole sums
    assert L.stmp_lstm_wide_rows_scratch_bytes(None) == 0
