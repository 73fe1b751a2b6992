"""The DyGrEncoder tutorial loop (examples/recurrent/dygrencoder_example.py) -- DyGrEncoder(C, L_g, aggr, H_h, L_l), ReLU, Linear(H_h, 1),
H and C carried from None (or from leaf H0 / C0, or None at every snapshot), a cumulative MSE divided by the number of snapshots and one
backward -- shared by tests/golden/make_goldens_dygrae.py, the CPU and GPU DyGrEncoder tests and tests/perf/bench_dygrae.py.

It also holds the float64 oracle.  `GatedGraphConv` restates PyG 2.x GatedGraphConv(out_channels, num_layers, aggr, bias=True) so the
unmodified reference dygrae.py can run on it; PyG is not installed where the goldens are made, so this restatement -- not an installed
PyG -- is the source of truth, written from PyG 2.x's source and not checked against an installed copy:
  * parameters: `weight` (num_layers, C, C), registered before `rnn` = torch.nn.GRUCell(C, C, bias);
  * draws: the GRUCell constructor's, then uniform(C, weight) = U(-1/sqrt(C), 1/sqrt(C)), then rnn.reset_parameters() draws all four GRU
    tensors again;
  * forward: more input channels than C raises ValueError, fewer are zero-padded to C; per layer m = x @ weight[l], m = aggr over the
    edges j -> i of w_e m_j (m_j without weights; no self loops added, duplicates kept), x = rnn(m, x);
  * add is a plain sum; mean the sum over the count of in-edges clamped to 1; max is new_zeros(N, C).scatter_reduce_(0, dst, msg, "amax",
    include_self=False): 0 for a node without in-edges, and on exact ties torch's amax backward splits the gradient evenly among the tied
    messages (counting the zero-initialised output as one more when the maximum is exactly 0).  PyG on CUDA with torch_scatter would
    instead route it to one arbitrary argmax.
`dygrae_step` is one DyGrEncoder step as a function of a parameter dict.  The fixture stores each case's description, the reference's
cost and fingerprints (tests/lstm64_seq.fingerprint); parameters come from the case's seed."""
import gzip
import io
import math
import os
import types

import torch

from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the tests)
from pytorch_geometric_temporal_b200.nn.recurrent import DyGrEncoder

FIXTURE = "dygrae.pt.gz"


def aggregate(m, edge_index, edge_weight, aggr):
    """PyG propagate of GatedGraphConv: aggr over the edges j -> i of w_e m_j."""
    src, dst = edge_index[0], edge_index[1]
    msg = m.index_select(0, src)
    if edge_weight is not None:
        msg = edge_weight.view(-1, 1).to(m.dtype) * msg
    if aggr == "max":
        return m.new_zeros(m.shape).scatter_reduce_(0, dst.view(-1, 1).expand_as(msg), msg, "amax", include_self=False)
    out = m.new_zeros(m.shape).index_add_(0, dst, msg)
    if aggr == "mean":
        cnt = m.new_zeros(m.size(0)).index_add_(0, dst, torch.ones_like(dst, dtype=m.dtype))
        out = out / cnt.clamp(min=1).unsqueeze(1)
    return out


def gru_cell(x, h, w_ih, w_hh, b_ih, b_hh):
    gi, gh = x @ w_ih.t() + b_ih, h @ w_hh.t() + b_hh
    ir, iz, inn = gi.chunk(3, 1)
    hr, hz, hn = gh.chunk(3, 1)
    r, z = torch.sigmoid(ir + hr), torch.sigmoid(iz + hz)
    n = torch.tanh(inn + r * hn)
    return (1 - z) * n + z * h


def ggc(p, x, edge_index, edge_weight, aggr, C):
    """GatedGraphConv from p = {weight, rnn.weight_ih, rnn.weight_hh, rnn.bias_ih, rnn.bias_hh}."""
    if x.size(-1) > C:
        raise ValueError("The number of input channels is not allowed to be larger than the number of output channels")
    if x.size(-1) < C:
        x = torch.cat([x, x.new_zeros(x.size(0), C - x.size(-1))], dim=1)
    for W in p["weight"]:
        x = gru_cell(aggregate(x @ W, edge_index, edge_weight, aggr), x, p["rnn.weight_ih"], p["rnn.weight_hh"], p["rnn.bias_ih"],
                     p["rnn.bias_hh"])
    return x


class GatedGraphConv(torch.nn.Module):
    """PyG 2.x GatedGraphConv in its parameter registration and draw order (see the module docstring)."""

    def __init__(self, out_channels, num_layers, aggr="add", bias=True, **kwargs):
        super().__init__()
        self.out_channels, self.num_layers, self.aggr = out_channels, num_layers, aggr
        self.weight = torch.nn.Parameter(torch.empty(num_layers, out_channels, out_channels))
        self.rnn = torch.nn.GRUCell(out_channels, out_channels, bias=bias)
        self.reset_parameters()

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.out_channels)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)
        self.rnn.reset_parameters()

    def forward(self, x, edge_index, edge_weight=None):
        p = {"weight": self.weight, **{f"rnn.{k}": v for k, v in self.rnn.named_parameters()}}
        return ggc(p, x, edge_index, edge_weight, self.aggr, self.out_channels)


def lstm_step(p, x, H, C, layers):
    """torch.nn.LSTM over one time step from p = {weight_ih_l{k}, ...}: (output (N, H_h), H (layers, N, H_h), C (layers, N, H_h))."""
    hs, cs = [], []
    for k in range(layers):
        g = x @ p[f"weight_ih_l{k}"].t() + p[f"bias_ih_l{k}"] + H[k] @ p[f"weight_hh_l{k}"].t() + p[f"bias_hh_l{k}"]
        i, f, gg, o = g.chunk(4, 1)
        c = torch.sigmoid(f) * C[k] + torch.sigmoid(i) * torch.tanh(gg)
        x = torch.sigmoid(o) * torch.tanh(c)
        hs.append(x)
        cs.append(c)
    return x, torch.stack(hs), torch.stack(cs)


def dygrae_step(p, c, x, edge_index, edge_weight, H=None, C=None):
    """One DyGrEncoder step of case c from the parameter dict p (keys conv_layer.*, recurrent_layer.*): (H_tilde, H, C), squeezed as the
    reference squeezes them."""
    conv = {k[len("conv_layer."):]: v for k, v in p.items() if k.startswith("conv_layer.")}
    lstm = {k[len("recurrent_layer."):]: v for k, v in p.items() if k.startswith("recurrent_layer.")}
    h = ggc(conv, x, edge_index, edge_weight, c["aggr"], c["C"])
    if (H is None) != (C is None):
        raise ValueError("Invalid hidden state and cell matrices.")
    if H is None:
        H = C = h.new_zeros(c["Ll"], h.size(0), c["Ho"])
    else:
        H, C = H[None, :, :], C[None, :, :]
        if H.dim() != 3:
            raise RuntimeError(f"expected a 3-D hidden state, got {H.dim()}-D")
    out, H, C = lstm_step(lstm, h, H, C, c["Ll"])
    return out.squeeze(), H.squeeze(), C.squeeze()


class RecurrentDyGr(torch.nn.Module):
    """The example's model (state_dict keys recurrent.*, linear.*); `cls` is this package's DyGrEncoder or the reference's."""

    def __init__(self, cls, C, Lg, aggr, Ho, Ll):
        super().__init__()
        self.recurrent = cls(C, Lg, aggr, Ho, Ll)
        self.linear = torch.nn.Linear(Ho, 1)


def carried_state(n, width, a, b, m):
    """A leaf state of exact multiples of 1/16 in [-0.5, 0.5], computed rather than stored."""
    i = torch.arange(n).unsqueeze(1) * a + torch.arange(width).unsqueeze(0) * b
    return ((i % m) - (m // 2)).float() / 16


def seeded_state(c):
    """The parameters of case c from its seed (float32 values): tensors with both trailing dimensions > 1 N(0, 1/fan), the rest N(0, 0.3),
    in sorted state_dict-key order."""
    keys = RecurrentDyGr(DyGrEncoder, c["C"], c["Lg"], c["aggr"], c["Ho"], c["Ll"]).state_dict()
    g = torch.Generator().manual_seed(c["seed"])
    state = {}
    for k in sorted(keys):
        shape = keys[k].shape
        scale = shape[-1] ** -0.5 if len(shape) >= 2 and min(shape[-2:]) > 1 else 0.3
        state[k] = (torch.randn(shape, generator=g, dtype=torch.float64) * scale).float()
    return state


def run(m, X, Y, ei, ew, H0=None, C0=None, carry=True):
    """(every step's prediction (S, N, 1), cost): H and C carried from H0 / C0 (carry) or None at every snapshot, cumulative MSE / S
    ((N, 1) - (N,) broadcasts, as in the example)."""
    h, c, cost, outs = H0, C0, 0, []
    for t in range(X.shape[0]):
        y, hn, cn = m.recurrent(X[t], ei, ew, h, c)
        if carry:
            h, c = hn, cn
        y = m.linear(torch.relu(y))
        outs.append(y)
        cost = cost + torch.mean((y - Y[t]) ** 2)
    return torch.stack(outs), cost / X.shape[0]


def load(golden_dir):
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def model_for(c, device="cpu", fused=True):
    m = RecurrentDyGr(DyGrEncoder, c["C"], c["Lg"], c["aggr"], c["Ho"], c["Ll"])
    m.load_state_dict(seeded_state(c))
    m.recurrent.fused_training = fused
    return m.to(device)


def states_for(c, n, device="cpu", dtype=torch.float32):
    """(H0, C0) leaves of a carried case, else (None, None)."""
    if c["state"] != "leaf":
        return None, None
    H0 = carried_state(n, c["Ho"], 7, 13, 17).to(device=device, dtype=dtype).requires_grad_(True)
    C0 = carried_state(n, c["Ho"], 5, 11, 19).to(device=device, dtype=dtype).requires_grad_(True)
    return H0, C0


def oracle_run(c, X, Y, ei, ew, H0=None, C0=None):
    """run() of case c in float64 on dygrae_step: (outs, cost, {parameter name: leaf})."""
    leaves = {k: v.double().to(X.device).requires_grad_(True) for k, v in seeded_state(c).items()}
    p = {k[len("recurrent."):]: v for k, v in leaves.items() if k.startswith("recurrent.")}
    m = types.SimpleNamespace(recurrent=lambda x, ei_, ew_, h, cc: dygrae_step(p, c, x, ei_, ew_, h, cc),
                              linear=lambda t: torch.nn.functional.linear(t, leaves["linear.weight"], leaves["linear.bias"]))
    outs, cost = run(m, X.double(), Y.double(), ei, None if ew is None else ew.double(), H0, C0, c["state"] != "none")
    return outs, cost, leaves


def check_reference(c, outs, cost, grads, gH0=None, gC0=None):
    """The float64 oracle's results of case c against the unmodified reference's fingerprints and exact cost."""
    cost = float(cost.detach())
    assert abs(cost - float(c["cost"])) <= 1e-10 * abs(float(c["cost"])), (cost, float(c["cost"]))
    got = {"out": outs, **{f"grad/{k}": v for k, v in grads.items()}}
    if gH0 is not None:
        got.update({"gH0": gH0, "gC0": gC0})
    assert sorted(got) == sorted(c["fingerprints"])
    for k, t in got.items():
        want = c["fingerprints"][k]
        assert torch.allclose(fingerprint(t), want, rtol=0, atol=1e-9 * float(want[-1]) + 1e-300), k
