"""AGCRN without a GPU: the op-for-op restatement against the unmodified reference bit for bit (K = 1's broadcast included), the
hand-written backward's algebra (agcrn.cu's decomposition, in float64 torch) against autograd, the state_dict keys and seeded
initialisation against the reference's, the reference's shape errors and the routing predicate with the library stubbed."""
import pytest
import torch

from oracle import refload
from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import AGCRN, AVWGCN
from pytorch_geometric_temporal_b200.nn.recurrent.agcrn import agcrn_cell

D = torch.float64
SHAPES = [(20, 8, 2, 1, 4), (20, 8, 2, 2, 4), (20, 8, 2, 3, 4), (13, 3, 5, 3, 6), (100, 64, 16, 2, 32), (7, 1, 1, 1, 1)]


def _ref_module():
    if not refload.available():
        pytest.skip("reference tree not present")
    return refload.load("nn.recurrent.agcrn")


def _inputs(N, cin, out, d, B=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, N, cin, generator=g, dtype=D), torch.randn(N, d, generator=g, dtype=D) * 0.7,
            torch.randn(B, N, out, generator=g, dtype=D))


def _params(m):
    return ((m._gate.weights_pool, m._gate.bias_pool, m.K), (m._update.weights_pool, m._update.bias_pool, m.K))


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("with_h", [False, True])
def test_restatement_matches_reference_bit_for_bit(shape, with_h):
    ref_mod = _ref_module()
    N, cin, out, K, d = shape
    torch.manual_seed(3)
    ref = ref_mod.AGCRN(*shape).to(D)
    with torch.no_grad():
        for p in ref.parameters():
            p.normal_(0, 0.3)
    X, E, H = _inputs(N, cin, out, d)
    H = H if with_h else None
    want = ref(X, E, H)
    got = agcrn_cell(X, E, H, *_params(ref), out)
    assert torch.equal(got, want)
    if K == 1:                               # the single weight block multiplies Y + S Y
        gate = ref._gate
        S = torch.softmax(torch.relu(E @ E.T), dim=1)
        Y = torch.cat((X, torch.zeros(*X.shape[:2], out, dtype=D) if H is None else H), dim=-1)
        W = torch.einsum("nd,dkio->nkio", E, gate.weights_pool)[:, 0]
        direct = torch.einsum("bni,nio->bno", Y + torch.einsum("nm,bmc->bnc", S, Y), W) + E @ gate.bias_pool
        assert torch.allclose(ref._gate(Y, E), direct, rtol=1e-12, atol=1e-12)


def hand_backward(X, E, H, gate, update, gh):
    """agcrn.cu's backward written out in float64 torch: the forward pieces as the kernels keep them (supports, node weights with their
    bias row, feature rows [slots | 1]), then k_agcrn_pw_update, dF / dW per node, the transposed support product, k_agcrn_pw_gate,
    the pools' gradients E^T [dW | db], dT, dS (K = 3 through T_2), the softmax and ReLU backward and dE."""
    (wp0, bp0, K), (wp1, bp1, _) = gate, update
    B, N, cin = X.shape
    out, d = gh.shape[2], E.shape[1]
    Ci, kci = cin + out, K * (cin + out)
    Hh = torch.zeros(B, N, out, dtype=D) if H is None else H
    A = E @ E.T
    S = torch.softmax(torch.relu(A), dim=1)
    T = [S] + ([2 * S @ S - torch.eye(N, dtype=D)] if K == 3 else [])
    slot = (lambda t: 0) if K == 1 else (lambda t: t + 1)
    pools = [torch.cat([wp.reshape(d, -1), bp], dim=1) for wp, bp in ((wp0, bp0), (wp1, bp1))]
    W = [(E @ p).view(N, kci + 1, -1) for p in pools]

    def feats(Y):
        P = [torch.einsum("nm,bmc->bnc", t, Y) for t in T]
        slots = [Y + P[0]] if K == 1 else [Y] + P
        return torch.cat(slots + [torch.ones(B, N, 1, dtype=D)], dim=-1)

    def supT(dF):
        dY = dF[..., :Ci].clone()
        for t, Tt in enumerate(T):
            dY = dY + torch.einsum("mn,bmc->bnc", Tt, dF[..., slot(t) * Ci:(slot(t) + 1) * Ci])
        return dY

    Y1 = torch.cat((X, Hh), dim=-1)
    F1 = feats(Y1)
    ZR = torch.sigmoid(torch.einsum("bnj,njo->bno", F1, W[0]))
    Z, R = ZR[..., :out], ZR[..., out:]
    Y2 = torch.cat((X, Z * Hh), dim=-1)
    F2 = feats(Y2)
    HC = torch.tanh(torch.einsum("bnj,njo->bno", F2, W[1]))

    dU = gh * (1 - R) * (1 - HC * HC)
    dF2 = torch.einsum("bno,njo->bnj", dU, W[1])[..., :kci]
    dW1 = torch.einsum("bnj,bno->njo", F2, dU)
    dY2 = supT(dF2)
    dZH = dY2[..., cin:]
    dG = torch.cat((dZH * Hh * (1 - Z) * Z, gh * (Hh - HC) * (1 - R) * R), dim=-1)
    dH = gh * R + dZH * Z
    dF1 = torch.einsum("bno,njo->bnj", dG, W[0])[..., :kci]
    dW0 = torch.einsum("bnj,bno->njo", F1, dG)
    dY1 = supT(dF1)
    dX = dY1[..., :cin] + dY2[..., :cin]
    dH = dH + dY1[..., cin:]
    dpool = [E.T @ dW.reshape(N, -1) for dW in (dW0, dW1)]
    grads_pool = []
    for dp, wp in zip(dpool, (wp0, wp1)):
        w = wp[0].numel()
        grads_pool += [dp[:, :w].view(wp.shape), dp[:, w:]]
    dT = [sum(dF1[b, :, slot(t) * Ci:(slot(t) + 1) * Ci] @ Y1[b].T + dF2[b, :, slot(t) * Ci:(slot(t) + 1) * Ci] @ Y2[b].T
              for b in range(B)) for t in range(len(T))]
    dS = dT[0] if K < 3 else dT[0] + 2 * (dT[1] @ S.T + S.T @ dT[1])
    dA = (torch.relu(A) > 0).to(D) * S * (dS - (dS * S).sum(1, keepdim=True))
    dE = dW0.reshape(N, -1) @ pools[0].T + dW1.reshape(N, -1) @ pools[1].T + (dA + dA.T) @ E
    return dX, dE, dH, *grads_pool


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("with_h", [False, True])
def test_backward_algebra_matches_autograd(shape, with_h):
    N, cin, out, K, d = shape
    torch.manual_seed(5)
    m = AGCRN(*shape).to(D)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.3)
    X, E, H = _inputs(N, cin, out, d, seed=1)
    H = H if with_h else None
    leaves = [t.clone().requires_grad_(True) if t is not None else None for t in (X, E, H)]
    gh = torch.randn(X.shape[0], N, out, generator=torch.Generator().manual_seed(2), dtype=D)
    y = agcrn_cell(*leaves, *_params(m), out)
    y.backward(gh)
    got = hand_backward(X, E, H, *_params(m), gh)
    want = [leaves[0].grad, leaves[1].grad, leaves[2].grad if with_h else None,
            m._gate.weights_pool.grad, m._gate.bias_pool.grad, m._update.weights_pool.grad, m._update.bias_pool.grad]
    for name, g, w in zip(("dX", "dE", "dH", "dwp_gate", "dbp_gate", "dwp_update", "dbp_update"), got, want):
        if w is None:
            continue
        assert torch.allclose(g, w, rtol=1e-10, atol=1e-12 * max(1.0, w.abs().max().item())), name


KEYS = ["_gate.weights_pool", "_gate.bias_pool", "_update.weights_pool", "_update.bias_pool"]


@pytest.mark.parametrize("shape", [(20, 8, 2, 2, 4), (100, 64, 16, 3, 32), (307, 1, 64, 2, 10), (5, 2, 3, 1, 1)])
def test_state_dict_and_seeded_init_match_reference(shape):
    ours = AGCRN(*shape)
    assert list(ours.state_dict()) == KEYS
    N, cin, out, K, d = shape
    assert (ours.number_of_nodes, ours.in_channels, ours.out_channels, ours.K, ours.embedding_dimensions) == shape
    assert ours._gate.weights_pool.shape == (d, K, cin + out, 2 * out) and ours._update.bias_pool.shape == (d, out)
    assert isinstance(ours._gate, AVWGCN) and ours._gate.K == K
    ref_mod = _ref_module()
    torch.manual_seed(11)
    ref = ref_mod.AGCRN(*shape)
    torch.manual_seed(11)
    ours = AGCRN(*shape)
    assert list(ref.state_dict()) == list(ours.state_dict())
    for k, v in ref.state_dict().items():
        assert torch.equal(v, ours.state_dict()[k]), k
    torch.manual_seed(12)
    ref_avw = ref_mod.AVWGCN(7, 3, K, d)
    torch.manual_seed(12)
    ours_avw = AVWGCN(7, 3, K, d)
    assert list(ref_avw.state_dict()) == list(ours_avw.state_dict()) == ["weights_pool", "bias_pool"]
    for k, v in ref_avw.state_dict().items():
        assert torch.equal(v, ours_avw.state_dict()[k]), k


@pytest.mark.parametrize("case", ["e_rows", "h_rows", "h_nodes", "h_channels", "h_2d"])
def test_shape_errors_raise_as_reference(case):
    m = AGCRN(6, 3, 2, 2, 4)
    X, E, H = torch.randn(2, 6, 3), torch.randn(6, 4), torch.randn(2, 6, 2)
    if case == "e_rows":
        E = torch.randn(5, 4)
    elif case == "h_rows":
        H = torch.randn(3, 6, 2)
    elif case == "h_nodes":
        H = torch.randn(2, 5, 2)
    elif case == "h_channels":
        H = torch.randn(2, 6, 3)
    else:
        H = torch.randn(6, 2)
    with pytest.raises(RuntimeError, match="AGCRN: "):       # raised before the CUDA check, so before any launch
        m(X, E, H)
    ref_mod = _ref_module()
    ref = ref_mod.AGCRN(6, 3, 2, 2, 4)
    with pytest.raises(RuntimeError):
        ref(X, E, H)


def _envelope(B, N, cin, out, K, d):
    return 0 <= B <= 8388607 and 1 <= N <= 4096 and cin >= 1 and 1 <= out <= 64 and cin + out <= 128 and 1 <= K <= 3 and 1 <= d <= 64


@pytest.mark.parametrize("shape,xdtype,edtype,hdtype,pdtype,needs_grad,fused_training,want", [
    ((20, 8, 2, 2, 4), torch.float32, torch.float32, None, torch.float32, False, True, True),
    ((20, 8, 2, 2, 4), torch.float32, torch.float32, torch.float32, torch.float32, True, True, True),
    ((20, 8, 2, 2, 4), torch.float32, torch.float32, None, torch.float32, True, False, False),
    ((20, 8, 2, 2, 4), torch.float32, torch.float32, None, torch.float32, False, False, True),
    ((20, 8, 2, 2, 4), torch.float64, torch.float32, None, torch.float32, False, True, False),
    ((20, 8, 2, 2, 4), torch.float32, torch.float64, None, torch.float32, False, True, False),
    ((20, 8, 2, 2, 4), torch.float32, torch.float32, torch.float64, torch.float32, False, True, False),
    ((20, 8, 2, 2, 4), torch.float32, torch.float32, None, torch.float64, False, True, False),
    ((20, 8, 2, 4, 4), torch.float32, torch.float32, None, torch.float32, False, True, False),
    ((20, 64, 65, 2, 4), torch.float32, torch.float32, None, torch.float32, False, True, False),
    ((20, 65, 64, 2, 4), torch.float32, torch.float32, None, torch.float32, False, True, False),
    ((20, 64, 64, 3, 64), torch.float32, torch.float32, None, torch.float32, False, True, True),
    ((20, 8, 2, 2, 65), torch.float32, torch.float32, None, torch.float32, False, True, False),
    ((4097, 1, 2, 2, 4), torch.float32, torch.float32, None, torch.float32, False, True, False),
    ((4096, 1, 2, 2, 4), torch.float32, torch.float32, None, torch.float32, False, True, True)])
def test_routing_predicate(monkeypatch, shape, xdtype, edtype, hdtype, pdtype, needs_grad, fused_training, want):
    monkeypatch.setattr(ops, "agcrn_supported", _envelope)
    N, cin, out, K, d = shape
    m = AGCRN(*shape).to(pdtype)
    m.fused_training = fused_training
    X, E = torch.zeros(2, N, cin, dtype=xdtype), torch.zeros(N, d, dtype=edtype)
    H = None if hdtype is None else torch.zeros(2, N, out, dtype=hdtype)
    assert m._fused_ok(X, E, H, needs_grad) is want
    assert m._fused_ok(torch.zeros(2, N, cin + 1), E, None, False) is False     # X's channels disagree with in_channels


def test_modules_refuse_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA only"):
        AGCRN(6, 3, 2, 2, 4)(torch.randn(2, 6, 3), torch.randn(6, 4))
    with pytest.raises(RuntimeError, match="CUDA only"):
        AVWGCN(5, 2, 2, 4)(torch.randn(2, 6, 5), torch.randn(6, 4))
