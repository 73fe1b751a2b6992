"""The LRGCN tutorial loop (examples/recurrent/lrgcn_example.py) -- LRGCN(F, out, R, B), ReLU, Linear(out, 1), H and C carried from None
(or from leaf H0 / C0), a cumulative MSE divided by the number of snapshots and one backward -- shared by
tests/golden/make_goldens_lrgcn.py, the CPU and GPU LRGCN tests and tests/perf/bench_lrgcn.py.

It also holds the float64 oracle: `RGCNConv` restates PyG RGCNConv's per-relation loop (aggr="mean", root weight, bias) as a module, so
the unmodified reference lrgcn.py can run on it, and `lrgcn_cell` is the same step as a function of a parameter dict.  The fixture stores
each case's description, the reference's cost and fingerprints (tests/lstm64_seq.fingerprint); parameters come from the case's seed."""
import gzip
import io
import math
import os
import types

import torch

from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the tests)
from pytorch_geometric_temporal_b200.nn.recurrent import LRGCN

FIXTURE = "lrgcn.pt.gz"


def _glorot(t):
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)


def relation_mean(x, edge_index, edge_type, r):
    """mean_r(x): per destination, the mean of x[src] over the edges src -> dst with edge_type == r (0 without such an edge)."""
    mask = edge_type == r
    src, dst = edge_index[0][mask], edge_index[1][mask]
    agg = torch.zeros_like(x).index_add_(0, dst, x[src])
    cnt = torch.zeros(x.size(0), dtype=x.dtype, device=x.device).index_add_(0, dst, torch.ones_like(dst, dtype=x.dtype))
    return agg / cnt.clamp(min=1).unsqueeze(1)


def rgcn(p, x, edge_index, edge_type, R):
    """RGCNConv(x) from its parameters p = {weight, comp (optional), root, bias}: sum_r mean_r(x) @ W_r + x @ root + bias."""
    W = p["weight"]
    if p.get("comp") is not None:
        W = (p["comp"] @ W.view(W.size(0), -1)).view(R, W.size(1), W.size(2))
    out = torch.zeros(x.size(0), W.size(2), dtype=x.dtype, device=x.device)
    for r in range(R):
        out = out + relation_mean(x, edge_index, edge_type, r) @ W[r]
    return out + x @ p["root"] + p["bias"]


class RGCNConv(torch.nn.Module):
    """PyG RGCNConv(in, out, num_relations, num_bases) on the per-relation loop path: parameters weight, comp, root, bias in PyG's
    registration and initialisation order."""

    def __init__(self, in_channels, out_channels, num_relations, num_bases=None, aggr="mean", root_weight=True, bias=True):
        super().__init__()
        assert aggr == "mean" and root_weight and bias
        self.num_relations = num_relations
        P = torch.nn.Parameter
        if num_bases is not None:
            self.weight = P(torch.empty(num_bases, in_channels, out_channels))
            self.comp = P(torch.empty(num_relations, num_bases))
        else:
            self.weight = P(torch.empty(num_relations, in_channels, out_channels))
            self.register_parameter("comp", None)
        self.root = P(torch.empty(in_channels, out_channels))
        self.bias = P(torch.empty(out_channels))
        _glorot(self.weight)
        if self.comp is not None:
            _glorot(self.comp)
        _glorot(self.root)
        torch.nn.init.zeros_(self.bias)

    def forward(self, x, edge_index, edge_type):
        return rgcn(dict(weight=self.weight, comp=self.comp, root=self.root, bias=self.bias), x, edge_index, edge_type, self.num_relations)


def lrgcn_cell(p, x, edge_index, edge_type, h, c, R):
    """One LRGCN step from the parameter dict p (keys conv_{x,h}_{g}.{weight,comp,root,bias}): (H', C')."""
    def conv(name, t):
        return rgcn({k: p.get(f"{name}.{k}") for k in ("weight", "comp", "root", "bias")}, t, edge_index, edge_type, R)

    def gate(g):
        return conv(f"conv_x_{g}", x) + conv(f"conv_h_{g}", h)
    I, F = torch.sigmoid(gate("i")), torch.sigmoid(gate("f"))
    cn = F * c + I * torch.tanh(gate("c"))
    O = torch.sigmoid(gate("o"))
    return O * torch.tanh(cn), cn


class RecurrentLRGCN(torch.nn.Module):
    """The example's model (state_dict keys recurrent.*, linear.*); `cls` is this package's LRGCN or the reference's."""

    def __init__(self, cls, F, out, R, B):
        super().__init__()
        self.recurrent = cls(F, out, R, B)
        self.linear = torch.nn.Linear(out, 1)


def carried_state(n, width, a, b, m):
    """A leaf state of exact multiples of 1/16 in [-0.5, 0.5], computed rather than stored."""
    i = torch.arange(n).unsqueeze(1) * a + torch.arange(width).unsqueeze(0) * b
    return ((i % m) - (m // 2)).float() / 16


def seeded_state(c):
    """The parameters of case c from its seed (float32 values): tensors with both trailing dimensions > 1 N(0, 1/fan), the rest N(0, 0.1),
    in sorted state_dict-key order."""
    keys = RecurrentLRGCN(LRGCN, c["F"], c["out"], c["R"], c["B"]).state_dict()
    g = torch.Generator().manual_seed(c["seed"])
    state = {}
    for k in sorted(keys):
        shape = keys[k].shape
        scale = shape[-1] ** -0.5 if len(shape) >= 2 and min(shape[-2:]) > 1 else 0.1
        state[k] = (torch.randn(shape, generator=g, dtype=torch.float64) * scale).float()
    return state


def edge_types(kind, edge_index, edge_weight):
    """The edge_type of a case: "attr" the example's float edge_attr (ones), "zero" all 0, "src_lt_dst" (src < dst) as int64."""
    if kind == "attr":
        return edge_weight
    if kind == "zero":
        return torch.zeros(edge_index.size(1), dtype=torch.int64, device=edge_index.device)
    return (edge_index[0] < edge_index[1]).to(torch.int64)


def run(m, X, Y, ei, et, H0=None, C0=None):
    """(every step's prediction (S, N, 1), cost): H and C carried from H0 / C0, cumulative MSE / S ((N, 1) - (N,) broadcasts, as in the
    example)."""
    h, c, cost, outs = H0, C0, 0, []
    for t in range(X.shape[0]):
        h, c = m.recurrent(X[t], ei, et, h, c)
        y = m.linear(torch.relu(h))
        outs.append(y)
        cost = cost + torch.mean((y - Y[t]) ** 2)
    return torch.stack(outs), cost / X.shape[0]


def load(golden_dir):
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def model_for(c, device="cpu", fused=True):
    m = RecurrentLRGCN(LRGCN, c["F"], c["out"], c["R"], c["B"])
    m.load_state_dict(seeded_state(c))
    m.recurrent.fused_training = fused
    return m.to(device)


def states_for(c, n, device="cpu", dtype=torch.float32):
    """(H0, C0) leaves of a carried case, else (None, None)."""
    if not c["carried"]:
        return None, None
    H0 = carried_state(n, c["out"], 7, 13, 17).to(device=device, dtype=dtype).requires_grad_(True)
    C0 = carried_state(n, c["out"], 5, 11, 19).to(device=device, dtype=dtype).requires_grad_(True)
    return H0, C0


def oracle_run(c, X, Y, ei, et, H0=None, C0=None):
    """run() of case c in float64 on lrgcn_cell: (outs, cost, {parameter name: leaf})."""
    leaves = {k: v.double().to(X.device).requires_grad_(True) for k, v in seeded_state(c).items()}
    p = {k[len("recurrent."):]: v for k, v in leaves.items() if k.startswith("recurrent.")}
    W = c["out"]

    def recurrent(x, ei_, et_, h, cc):
        z = torch.zeros(x.size(0), W, dtype=torch.float64, device=x.device)
        return lrgcn_cell(p, x, ei_, et_, z if h is None else h, z if cc is None else cc, c["R"])
    m = types.SimpleNamespace(recurrent=recurrent,
                              linear=lambda t: torch.nn.functional.linear(t, leaves["linear.weight"], leaves["linear.bias"]))
    outs, cost = run(m, X.double(), Y.double(), ei, et, H0, C0)
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
