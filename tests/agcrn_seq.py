"""The AGCRN cases (examples/recurrent/agcrn_example.py's epoch, the reference's unit-test shape and the paper's two stacked layers),
shared by tests/golden/make_goldens_agcrn.py, the CPU and GPU AGCRN tests and tests/perf/bench_agcrn.py.

Every case is a Net of one or two AGCRN layers sharing one embedding E, with an optional Linear head, run by `run`:
* tutorial   AGCRN(20, 8, 2, K, 4), ReLU, Linear(2, 1) over the 102 chickenpox training snapshots at lags 8, h carried across them without a
             detach, the cumulative MSE / 102 and one backward, exactly as the example writes its epoch; E xavier-uniform (trained or not)
* unit       AGCRN(100, 64, 16, K, 32) on one (1, 100, 64) snapshot: H = layer(X, E), then layer(X, E, H), as the reference's unit test;
             the cost is a fixed random projection of the last H
* paper      AGCRN(307, 1, 64, 2, 10) and AGCRN(307, 64, 64, 2, 10) over T = 12 steps of B = 4 windows (pems04_like's 307 nodes), then
             Linear(64, 1) against a random target
The parameters, E and the inputs come from the case's seed as float32 values, so a float64 run and a float32 run see the same numbers."""
import math
import os

import torch

from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the tests)

FIXTURE = "agcrn.pt.gz"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = {
    "tutorial": dict(kind="tutorial", K=2, train_e=False, seed=501),
    "tutorial_e": dict(kind="tutorial", K=2, train_e=True, seed=502),
    "k1": dict(kind="tutorial", K=1, train_e=True, seed=503),
    "k3": dict(kind="tutorial", K=3, train_e=True, seed=504),
    "unit_k2": dict(kind="unit", K=2, train_e=True, seed=505),
    "unit_k3": dict(kind="unit", K=3, train_e=True, seed=506),
    "paper": dict(kind="paper", K=2, train_e=True, seed=507),
}


def layer_shapes(c):
    """[(number_of_nodes, in_channels, out_channels, K, embedding_dimensions)] of case c's layers, and its head's width (or None)."""
    if c["kind"] == "tutorial":
        return [(20, 8, 2, c["K"], 4)], 2
    if c["kind"] == "unit":
        return [(100, 64, 16, c["K"], 32)], None
    return [(307, 1, 64, c["K"], 10), (307, 64, 64, c["K"], 10)], 64


class Net(torch.nn.Module):
    """The case's AGCRN layers (`layers.<i>.*` keys) and head (`linear.*`)."""

    def __init__(self, cls, c):
        super().__init__()
        shapes, head = layer_shapes(c)
        self.layers = torch.nn.ModuleList(cls(*s) for s in shapes)
        self.linear = torch.nn.Linear(head, 1) if head else None


def seeded_state(c, cls):
    """The parameters of case c from its seed (float32 values): weights_pool N(0, 2 / (in + out)), everything else N(0, 0.3), in sorted
    key order."""
    m = Net(cls, c)
    g = torch.Generator().manual_seed(c["seed"])
    state = dict(m.state_dict())
    for k in sorted(state):
        shape = state[k].shape
        scale = math.sqrt(2.0 / (shape[-2] + shape[-1])) if k.endswith("weights_pool") else 0.3
        state[k] = (torch.randn(shape, generator=g, dtype=torch.float64) * scale).float()
    return state


def chickenpox(lags=8, train_ratio=0.2):
    """(X (S, 20, lags), Y (S, 20)) of temporal_signal_split(ChickenpoxDatasetLoader().get_dataset(lags), 0.2)'s training part."""
    import numpy as np
    z = np.load(os.path.join(ROOT, "pytorch_geometric_temporal_b200", "dataset", "data", "chickenpox.npz"))
    FX = np.asarray(z["FX"], dtype=np.float32)
    n = FX.shape[0] - lags
    S = int(train_ratio * n)
    X = torch.from_numpy(np.stack([FX[i:i + lags].T for i in range(n)]).copy())
    Y = torch.from_numpy(np.stack([FX[i + lags] for i in range(n)]).copy())
    return X[:S], Y[:S]


def inputs(c):
    """(E, X, Y) of case c as float32: tutorial X (102, 1, 20, 8) and Y (102, 20); unit X (1, 100, 64), Y a (1, 100, 16) projection;
    paper X (4, 12, 307, 1), Y (4, 307, 1)."""
    g = torch.Generator().manual_seed(c["seed"] + 1000)
    (N, _, _, _, d), = layer_shapes(c)[0][:1]
    if c["kind"] == "tutorial":
        E = torch.empty(N, d, dtype=torch.float32)
        torch.nn.init.xavier_uniform_(E, generator=g)
        X, Y = chickenpox()
        return E, X.view(-1, 1, 20, 8), Y
    f32 = dict(generator=g, dtype=torch.float32)
    E = torch.randn(N, d, **f32)
    if c["kind"] == "unit":
        return E, torch.rand(1, 100, 64, **f32) * 2 - 1, torch.randn(1, 100, 16, **f32)
    return E, torch.randn(4, 12, 307, 1, **f32), torch.randn(4, 307, 1, **f32)


def model_for(c, cls, device, dtype):
    m = Net(cls, c)
    m.load_state_dict(seeded_state(c, cls))
    return m.to(device=device, dtype=dtype)


def run(m, c, device, dtype, retain=False):
    """One forward and backward of case c on model m.  -> (outputs, cost, {gradient name: tensor}): the parameters' gradients under their
    keys, E's (when trained) and X's (unit and paper) under "E" and "X"."""
    E, X, Y = (t.to(device=device, dtype=dtype) for t in inputs(c))
    if c["train_e"]:
        E.requires_grad_(True)
    layers = list(m.layers)
    if c["kind"] == "tutorial":
        h, outs, cost = None, [], 0
        for t in range(X.shape[0]):
            h = layers[0](X[t], E, h)
            y = m.linear(torch.relu(h))
            outs.append(y)
            cost = cost + torch.mean((y - Y[t].view(1, 20, 1)) ** 2)
        cost = cost / X.shape[0]
        out = torch.stack(outs)
    elif c["kind"] == "unit":
        X.requires_grad_(True)
        H = layers[0](X, E)
        out = layers[0](X, E, H)
        cost = (out * Y).sum()
    else:
        X.requires_grad_(True)
        h1 = h2 = None
        for t in range(X.shape[1]):
            h1 = layers[0](X[:, t], E, h1)
            h2 = layers[1](h1, E, h2)
        out = m.linear(h2)
        cost = torch.mean((out - Y) ** 2)
    cost.backward(retain_graph=retain)
    grads = {k: p.grad for k, p in m.named_parameters()}
    if c["train_e"]:
        grads["E"] = E.grad
    if X.requires_grad:
        grads["X"] = X.grad
    return out.detach(), cost.detach(), grads


def reference_class():
    """The unmodified reference AGCRN on oracle/stubs."""
    from oracle import refload
    return refload.load("nn.recurrent.agcrn").AGCRN


def load(golden_dir):
    import gzip
    import io
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)
