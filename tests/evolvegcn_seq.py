"""The EvolveGCN tutorial loops (examples/recurrent/evolvegcno_example.py, evolvegcnh_example.py) -- EvolveGCNO(C) or EvolveGCNH(nodes, C),
ReLU, Linear(C, 1), the weight carried across snapshots, a cumulative MSE divided by the number of snapshots ((N, 1) - (N,) broadcasts, as
in the examples), one backward per epoch and `weight = weight.detach()` between epochs -- shared by tests/golden/make_goldens_evolvegcn.py,
the CPU and GPU EvolveGCN tests and tests/perf/bench_evolvegcn.py.

It also holds the float64 oracle and the PyG pieces the unmodified reference needs on top of oracle/stubs:
  * `TopKPooling` restates PyG 2.x TopKPooling(in_channels, ratio) -- PyG is not installed where the goldens are made, so this restatement,
    written from PyG 2.x's source and not checked against an installed copy, is the source of truth: `select.weight` (1, C) drawn
    U(-1/sqrt(C), 1/sqrt(C)) by SelectTopK's constructor and again by TopKPooling's reset_parameters; s = tanh((x * w).sum(-1) / |w|);
    k = int(ratio) when ratio >= 1, else ceil(float(ratio) * N) in s's dtype; perm = the first k of a stable descending sort of s; the
    result's first element is x[perm] * s[perm];
  * gcn_norm is oracle.pyg.gcn_norm with PyG's dtype default (ones of the default dtype when edge_weight is None);
  * torch_geometric.typing gets the names Adj and SparseTensor.
`egcn_step` is one step as a function of a parameter dict; `oracle_run` the tutorial loop on it."""
import gzip
import io
import math
import os
import sys
import types

import torch

from dygrae_seq import gru_cell
from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the tests)
from oracle import pyg
from pytorch_geometric_temporal_b200.nn.recurrent import EvolveGCNH, EvolveGCNO

FIXTURE = "evolvegcn.pt.gz"


def topk_k(ratio, n, dtype):
    if ratio >= 1:
        return min(int(ratio), n)
    return min(int((float(ratio) * torch.tensor([n], dtype=dtype)).ceil()), n)


class TopKPooling(torch.nn.Module):
    """PyG 2.x TopKPooling (see the module docstring); returns (x, edge_index, edge_attr, batch, perm, score[perm]) as PyG does, the edge
    filtering left out (EvolveGCNH reads only the first element)."""

    def __init__(self, in_channels, ratio=0.5, min_score=None, multiplier=1.0, nonlinearity="tanh"):
        super().__init__()
        self.in_channels, self.ratio = in_channels, ratio
        self.select = torch.nn.Module()
        self.select.weight = torch.nn.Parameter(torch.empty(1, in_channels))
        self._draw()
        self.reset_parameters()

    def _draw(self):
        bound = 1.0 / math.sqrt(self.in_channels)
        with torch.no_grad():
            self.select.weight.uniform_(-bound, bound)

    def reset_parameters(self):
        self._draw()

    def forward(self, x, edge_index, edge_attr=None, batch=None, attn=None):
        X, perm, s = topk_pool(x, self.select.weight, self.ratio)
        return X, edge_index, edge_attr, batch, perm, s


def topk_pool(x, w, ratio):
    score = torch.tanh((x * w).sum(dim=-1) / w.norm(p=2, dim=-1))
    k = topk_k(ratio, x.size(0), score.dtype)
    perm = torch.sort(score, descending=True, stable=True).indices[:k]
    return x[perm] * score[perm].view(-1, 1), perm, score[perm]


def gcn_norm(edge_index, edge_weight=None, num_nodes=None, improved=False, add_self_loops=True, flow="source_to_target", dtype=None):
    return pyg.gcn_norm(edge_index, edge_weight, num_nodes, improved, add_self_loops, torch.get_default_dtype() if dtype is None else dtype)


def reference_classes():
    """(EvolveGCNO, EvolveGCNH) of the unmodified reference on oracle/stubs plus the pieces above."""
    from oracle import refload
    sys.path.insert(0, refload._STUBS)
    import torch_geometric.nn as tgnn
    import torch_geometric.typing as tgt
    tgt.Adj = torch.Tensor
    tgt.SparseTensor = type("SparseTensor", (), {})
    tgnn.TopKPooling = TopKPooling
    gc = types.ModuleType("torch_geometric.nn.conv.gcn_conv")
    gc.gcn_norm = gcn_norm
    sys.modules["torch_geometric.nn.conv.gcn_conv"] = gc
    o = refload.load("nn.recurrent.evolvegcno").EvolveGCNO
    h = refload.load("nn.recurrent.evolvegcnh").EvolveGCNH
    return o, h


def make_recurrent(cls_o, cls_h, c):
    flags = dict(improved=c["improved"], normalize=c["normalize"], add_self_loops=c["loops"])
    return cls_h(c["nodes"], c["C"], **flags) if c["kind"] == "H" else cls_o(c["C"], **flags)


class RecurrentEGCN(torch.nn.Module):
    """The examples' model (state_dict keys recurrent.*, linear.*)."""

    def __init__(self, recurrent, C):
        super().__init__()
        self.recurrent = recurrent
        self.linear = torch.nn.Linear(C, 1)


def seeded_state(c):
    """The parameters of case c from its seed (float32 values): tensors with both trailing dimensions > 1 N(0, 1/fan), the rest N(0, 0.3),
    in sorted state_dict-key order."""
    keys = RecurrentEGCN(make_recurrent(EvolveGCNO, EvolveGCNH, c), c["C"]).state_dict()
    g = torch.Generator().manual_seed(c["seed"])
    state = {}
    for k in sorted(keys):
        shape = keys[k].shape
        scale = shape[-1] ** -0.5 if len(shape) >= 2 and min(shape[-2:]) > 1 else 0.3
        state[k] = (torch.randn(shape, generator=g, dtype=torch.float64) * scale).float()
    return state


def model_for(c, device="cpu", fused=True):
    m = RecurrentEGCN(make_recurrent(EvolveGCNO, EvolveGCNH, c), c["C"])
    m.load_state_dict(seeded_state(c))
    m.recurrent.fused_training = fused
    return m.to(device)


def run(m, X, Y, ei, ew, epochs=1, retain=False):
    """The examples' training loop without the optimizer: per epoch the snapshots' cumulative MSE / S and one backward (retain_graph as
    the -O example), then `weight = weight.detach()`; gradients accumulate over the epochs.  (every step's prediction of the last epoch
    (S, N, 1), the last epoch's cost)."""
    for _ in range(epochs):
        cost, outs = 0, []
        for t in range(X.shape[0]):
            y = m.linear(torch.relu(m.recurrent(X[t], ei, ew)))
            outs.append(y)
            cost = cost + torch.mean((y - Y[t]) ** 2)
        cost = cost / X.shape[0]
        cost.backward(retain_graph=retain)
        m.recurrent.weight = m.recurrent.weight.detach()
    return torch.stack(outs), cost


def conv(W, x, ei, ew, c):
    """GCNConv_Fixed_W: Op (x W)."""
    if c["normalize"]:
        ei, ew = pyg.gcn_norm(ei, ew, x.size(0), c["improved"], c["loops"], x.dtype)
    xw = x @ W
    msg = xw.index_select(0, ei[0])
    if ew is not None:
        msg = ew.view(-1, 1).to(xw.dtype) * msg
    return xw.new_zeros(xw.shape).index_add(0, ei[1], msg)


def egcn_step(p, c, W_prev, x, ei, ew):
    """One step of case c from the parameter dict p (keys initial_weight, recurrent_layer.*, pooling_layer.select.weight): (out, W_new),
    W_prev (C, C) or None (initial_weight)."""
    W_prev = p["initial_weight"][0] if W_prev is None else W_prev
    g = [p[f"recurrent_layer.{k}_l0"] for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    if c["kind"] == "H":
        xt = topk_pool(x, p["pooling_layer.select.weight"], c["C"] / c["nodes"])[0]
        if xt.size(0) != c["C"]:
            raise RuntimeError(f"input batch {xt.size(0)} != hidden batch {c['C']}")
        W = gru_cell(xt, W_prev, *g)
    else:
        W = gru_cell(W_prev, W_prev, *g)
    return conv(W, x, ei, ew, c), W


def oracle_run(c, X, Y, ei, ew, epochs=1):
    """run() of case c in float64 on egcn_step: (outs, cost, {parameter name: leaf})."""
    leaves = {k: v.double().to(X.device).requires_grad_(True) for k, v in seeded_state(c).items()}
    p = {k[len("recurrent."):]: v for k, v in leaves.items() if k.startswith("recurrent.")}

    class Rec:
        weight = None

        def __call__(self, x, ei_, ew_):
            out, W = egcn_step(p, c, None if self.weight is None else self.weight[0], x, ei_, ew_)
            self.weight = W[None]
            return out
    m = types.SimpleNamespace(recurrent=Rec(), linear=lambda t: torch.nn.functional.linear(t, leaves["linear.weight"], leaves["linear.bias"]))
    outs, cost = run(m, X.double(), Y.double(), ei, None if ew is None else ew.double(), epochs, retain=True)
    return outs, cost, leaves


def load(golden_dir):
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def graph_of(c, golden_dir):
    """(edge_index, edge_weight or None, X (S, N, C), Y (S, N)) of case c."""
    from gconvgru_seq import chickenpox_train_split
    from wikimaths_seq import load as load_wikimaths
    if c["graph"] == "chickenpox":
        ei, ew, X, Y = chickenpox_train_split()
    elif c["graph"] == "wikimaths":
        w = load_wikimaths(golden_dir)
        ei, ew, X, Y = w["edge_index"], w["edge_weight"], w["X"], w["Y"]
    else:                                    # the reference's unit-test shape: 100 nodes, 8 channels, a seeded random weighted graph
        g = torch.Generator().manual_seed(c["seed"])
        ei = torch.randint(0, 100, (2, 400), generator=g)
        f32 = dict(generator=g, dtype=torch.float32)
        ew = torch.rand(400, **f32)
        X, Y = torch.randn(5, 100, 8, **f32), torch.randn(5, 100, **f32)
    return ei, (ew if c["weights"] else None), X, Y


def check_reference(c, outs, cost, grads):
    """The float64 oracle's results of case c against the unmodified reference's fingerprints and exact cost."""
    cost = float(cost.detach())
    assert abs(cost - float(c["cost"])) <= 1e-10 * abs(float(c["cost"])), (cost, float(c["cost"]))
    got = {"out": outs, **{f"grad/{k}": v for k, v in grads.items()}}
    assert sorted(got) == sorted(c["fingerprints"])
    for k, t in got.items():
        want = c["fingerprints"][k]
        assert torch.allclose(fingerprint(t), want, rtol=0, atol=1e-9 * float(want[-1]) + 1e-300), k
