"""The MPNN-LSTM tutorial loop (examples/recurrent/mpnnlstm_example.py) -- MPNNLSTM, ReLU, Linear(2*32 + in + window - 1, 1), a cumulative
MSE divided by the number of snapshots ((M, 1) - (M,) broadcasts, as in the example), one backward per epoch, an optional eval pass --
shared by tests/golden/make_goldens_mpnnlstm.py, the CPU and GPU MPNN-LSTM tests and tests/perf/bench_mpnnlstm.py.

Dropout masks: every training call with p > 0 draws u = torch.rand(2, R, 32) from the case's own generator (layer 1, then layer 2) and
keeps an element where u >= p.  The unmodified reference module gets them through a replaced `F` (its relu is torch's, its dropout reads
the next u); this package's module through `_uniforms`.  `mpnn_forward` is the float64 restatement of one call as a function of a
parameter dict and a buffer dict (BatchNorm's running statistics, updated in training mode); `oracle_run` is the loop on it."""
import gzip
import io
import os
import types

import numpy as np
import torch

from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the tests)
from oracle import pyg
from pytorch_geometric_temporal_b200.nn.recurrent import MPNNLSTM

FIXTURE = "mpnnlstm.pt.gz"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Masks:
    """The dropout uniforms of a case: one (2, R, 32) draw per training call from a generator seeded with the case's seed."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def draw(self, R):
        return torch.rand(2, R, 32, generator=self.g, dtype=torch.float32)


def reference_class(masks):
    """The unmodified reference MPNNLSTM on oracle/stubs, its F replaced so that dropout takes the masks of `masks`."""
    from oracle import refload
    mod = refload.load("nn.recurrent.mpnn_lstm")
    state = {}

    def dropout(X, p, training):
        if not training or p == 0:
            return X
        if state.get("layer", 0) == 0:
            state["u"] = masks.draw(X.size(0))
        layer = state.get("layer", 0)
        state["layer"] = 1 - layer
        return X * (state["u"][layer] >= p).to(X.dtype) / (1 - p)
    mod.F = types.SimpleNamespace(relu=torch.nn.functional.relu, dropout=dropout)
    return mod.MPNNLSTM


class RecurrentMPNN(torch.nn.Module):
    """The example's model (state_dict keys recurrent.*, linear.*)."""

    def __init__(self, recurrent, width):
        super().__init__()
        self.recurrent = recurrent
        self.linear = torch.nn.Linear(width, 1)

    def forward(self, x, ei, ew):
        return self.linear(torch.relu(self.recurrent(x, ei, ew)))


def width(c):
    return 2 * 32 + c["cin"] + c["window"] - 1


def make(cls, c):
    r = cls(c["cin"], 32, c["nodes"], c["window"], c["p"])
    if c["momentum"] != "default":
        r._batch_norm_1.momentum = r._batch_norm_2.momentum = c["momentum"]
    return RecurrentMPNN(r, width(c))


def seeded_state(c):
    """The parameters of case c from its seed (float32 values): tensors with both trailing dimensions > 1 N(0, 1/fan), the rest N(0, 0.3)
    (BatchNorm's weight 1 + N(0, 0.3)), in sorted key order; the buffers at their initial values."""
    m = make(MPNNLSTM, c)
    g = torch.Generator().manual_seed(c["seed"])
    state = dict(m.state_dict())
    for k in sorted(k for k, _ in m.named_parameters()):
        shape = state[k].shape
        scale = shape[-1] ** -0.5 if len(shape) >= 2 and min(shape[-2:]) > 1 else 0.3
        state[k] = (torch.randn(shape, generator=g, dtype=torch.float64) * scale + (1.0 if "_batch_norm" in k and k.endswith("weight")
                                                                                       else 0.0)).float()
    return state


def model_for(c, device="cpu"):
    m = make(MPNNLSTM, c)
    m.load_state_dict(seeded_state(c))
    masks = Masks(c["seed"])
    m.recurrent._uniforms = lambda R, dev: masks.draw(R).to(dev)
    return m.to(device)


def chickenpox(lags=4, train_ratio=0.2):
    """(edge_index, edge_weight, (X, Y) of the train split, (X, Y) of the test split) of temporal_signal_split(dataset, 0.2) of the in-tree
    chickenpox data (ChickenpoxDatasetLoader().get_dataset(lags))."""
    z = np.load(os.path.join(ROOT, "pytorch_geometric_temporal_b200", "dataset", "data", "chickenpox.npz"))
    ei = torch.tensor(z["edges"], dtype=torch.int64).T.contiguous()
    FX = np.asarray(z["FX"], dtype=np.float32)
    n = FX.shape[0] - lags
    S = int(train_ratio * n)
    X = torch.from_numpy(np.stack([FX[i:i + lags].T for i in range(n)]).copy())
    Y = torch.from_numpy(np.stack([FX[i + lags] for i in range(n)]).copy())
    return ei, torch.ones(ei.shape[1]), (X[:S], Y[:S]), (X[S:], Y[S:])


def graph_of(c, golden_dir):
    """(edge_index, edge_weight or None, (X (S, R, cin), Y (S, M)) train, (X, Y) eval or None) of case c."""
    ev = None
    if c["graph"] == "chickenpox":
        ei, ew, (X, Y), test = chickenpox()
        if c["window"] == 4:                 # the four lags as 80 x 1 rows: row t * 20 + n = lag t of node n
            X = X.transpose(1, 2).reshape(X.shape[0], 80, 1)
        elif c["window"] == 2:               # B = 2, window = 2: snapshots s .. s + 3 stacked, each (20, 4)
            X = torch.stack([X[s:s + 4].reshape(80, 4) for s in range(20)])
            Y = torch.stack([Y[s:s + 2].reshape(40) for s in range(20)])
        if c["eval"]:
            ev = test
    elif c["graph"] == "wikimaths":
        from wikimaths_seq import load as load_wikimaths
        w = load_wikimaths(golden_dir)
        ei, ew, X, Y = w["edge_index"], w["edge_weight"], w["X"], w["Y"]
    else:                                    # the reference's unit-test shape: 100 nodes, 64 features, a seeded random weighted graph
        g = torch.Generator().manual_seed(c["seed"])
        ei = torch.randint(0, 100, (2, 1000), generator=g)
        f32 = dict(generator=g, dtype=torch.float32)
        ew = torch.rand(1000, **f32)
        X, Y = torch.rand(5, 100, 64, **f32) * 2 - 1, torch.randn(5, 100, **f32)
    return ei, (ew if c["weights"] else None), (X, Y), ev


def run(m, train, ev, ei, ew, epochs=1, retain=False):
    """The example's loop without the optimizer: per epoch the snapshots' cumulative MSE / S and one backward (gradients accumulate), then
    with `ev` an eval pass.  (every prediction of the last epoch (S, M, 1), its cost, the eval predictions or None)."""
    X, Y = train
    m.train()
    for _ in range(epochs):
        cost, outs = 0, []
        for t in range(X.shape[0]):
            y = m(X[t], ei, ew)
            outs.append(y)
            cost = cost + torch.mean((y - Y[t]) ** 2)
        cost = cost / X.shape[0]
        cost.backward(retain_graph=retain)
    evs = None
    if ev is not None:
        m.eval()
        with torch.no_grad():
            evs = torch.stack([m(x, ei, ew) for x in ev[0]])
    return torch.stack(outs), cost, evs


# ---- the float64 restatement ----------------------------------------------------------------------------------------------------------
def _bn(x, P, B, k, training, momentum):
    w, b = P[f"{k}.weight"], P[f"{k}.bias"]
    if not training:
        return (x - B[f"{k}.running_mean"]) / torch.sqrt(B[f"{k}.running_var"] + 1e-5) * w + b
    mean, var = x.mean(0), x.var(0, unbiased=False)
    with torch.no_grad():
        B[f"{k}.num_batches_tracked"] += 1
        mom = 1.0 / float(B[f"{k}.num_batches_tracked"]) if momentum is None else momentum
        B[f"{k}.running_mean"] = (1 - mom) * B[f"{k}.running_mean"] + mom * mean.detach()
        B[f"{k}.running_var"] = (1 - mom) * B[f"{k}.running_var"] + mom * x.detach().var(0, unbiased=True)
    return (x - mean) / torch.sqrt(var + 1e-5) * w + b


def _lstm(xs, P, k):
    wi, wh, bi, bh = (P[f"{k}.{n}_l0"] for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
    h = c = xs.new_zeros(xs.shape[1], wh.shape[1])
    hs = []
    for x in xs:
        i, f, g, o = (x @ wi.T + bi + h @ wh.T + bh).chunk(4, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        hs.append(h)
    return torch.stack(hs), h


def mpnn_forward(P, B, c, X, ei, ew, u, training, momentum=0.1):
    """One MPNNLSTM call of case c in X's dtype from parameters P and buffers B (keys without the `recurrent.` prefix); u (2, R, 32) or
    None.  B is updated in training mode."""
    T, N, F = c["window"], c["nodes"], c["cin"]
    S = X.view(-1, T, N, F).transpose(1, 2).reshape(-1, T, F)
    S = torch.cat([S[:, 0, :]] + [S[:, t, F - 1].unsqueeze(1) for t in range(1, T)], dim=1)
    e, w = pyg.gcn_norm(ei, ew, X.size(0), False, True, X.dtype)
    Z, h = [], X
    for layer in (1, 2):
        xw = h @ P[f"_convolution_{layer}.lin.weight"].T
        y = xw.new_zeros(xw.shape).index_add(0, e[1], w.view(-1, 1) * xw.index_select(0, e[0])) + P[f"_convolution_{layer}.bias"]
        h = _bn(torch.relu(y), P, B, f"_batch_norm_{layer}", training, momentum)
        if u is not None:
            h = h * (u[layer - 1] >= c["p"]).to(h.dtype) / (1 - c["p"])
        Z.append(h)
    H = torch.cat(Z, dim=1)
    H = H.view(-1, T, N, H.size(1)).transpose(0, 1).contiguous().view(T, -1, H.size(1))
    seq, h1 = _lstm(H, P, "_recurrent_1")
    _, h2 = _lstm(seq, P, "_recurrent_2")
    return torch.cat([h1, h2, S], dim=1)


def oracle_run(c, train, ev, ei, ew, epochs=1):
    """run() of case c in float64 on mpnn_forward: (outs, cost, evs, {parameter name: leaf}, {buffer name: value})."""
    state = seeded_state(c)
    m0 = make(MPNNLSTM, c)
    pnames = {k for k, _ in m0.named_parameters()}
    leaves = {k: v.double().requires_grad_(True) for k, v in state.items() if k in pnames}
    bufs = {k[len("recurrent."):]: v.double() if v.is_floating_point() else v.clone() for k, v in state.items() if k not in pnames}
    P = {k[len("recurrent."):]: v for k, v in leaves.items() if k.startswith("recurrent.")}
    masks = Masks(c["seed"])
    mom = None if c["momentum"] is None else (0.1 if c["momentum"] == "default" else c["momentum"])

    class Model:
        training = True

        def train(self):
            self.training = True

        def eval(self):
            self.training = False

        def __call__(self, x, ei_, ew_):
            u = masks.draw(x.size(0)).double() if self.training and c["p"] > 0 else None
            h = mpnn_forward(P, bufs, c, x, ei_, ew_, u, self.training, mom)
            return torch.nn.functional.linear(torch.relu(h), leaves["linear.weight"], leaves["linear.bias"])
    dw = lambda t: None if t is None else t.double()
    outs, cost, evs = run(Model(), (train[0].double(), train[1].double()), None if ev is None else (ev[0].double(), ev[1].double()), ei,
                          dw(ew), epochs, retain=True)
    return outs, cost, evs, leaves, {f"recurrent.{k}": v for k, v in bufs.items()}


def load(golden_dir):
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def results(outs, cost, evs, grads, bufs):
    """The quantities a golden case records: fingerprints of the outputs, eval outputs, every parameter gradient and running statistic."""
    got = {"out": outs, **{f"grad/{k}": v for k, v in grads.items()}, **{f"buf/{k}": v.double() for k, v in bufs.items()}}
    if evs is not None:
        got["eval"] = evs
    return got


def check_reference(c, outs, cost, evs, grads, bufs):
    """The float64 oracle's results of case c against the unmodified reference's fingerprints and exact cost."""
    cost = float(cost.detach())
    assert abs(cost - float(c["cost"])) <= 1e-10 * abs(float(c["cost"])), (cost, float(c["cost"]))
    got = results(outs, cost, evs, grads, bufs)
    assert sorted(got) == sorted(c["fingerprints"])
    for k, t in got.items():
        want = c["fingerprints"][k]
        assert torch.allclose(fingerprint(t), want, rtol=0, atol=1e-9 * float(want[-1]) + 1e-300), k
