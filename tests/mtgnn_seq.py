"""The MTGNN cases, shared by tests/golden/make_goldens_mtgnn.py, the CPU and GPU MTGNN tests and tests/perf/bench_mtgnn.py.

Every case builds MTGNN with the reference test's hyper-parameters (207 nodes, k = 20, node_dim 40, conv / residual channels 32, skip
64, end 128, in_dim 2, 3 layers, kernel set 2/3/6/7, propalpha 0.05, tanhalpha 3) unless it says otherwise, draws the parameters
from its seed and runs two training steps (MAE against a fixed target, backward, Adam at lr 1e-4) at dropout 0, then one eval call:
* idx        a permutation idx of the nodes, the input permuted alike (the reference test's first model)
* fe         static features FE with xd = 8 (nodevec2 is nodevec1)
* predef     build_adj = False with a predefined random graph of about ten edges per node (the reference's BA-graph A_tilde)
* nogcn_dil2 gcn_true = False, dilation_exponential = 2, non-affine LayerNorm
* seq24      24 input steps (above the receptive field 19), out_dim 5, non-affine LayerNorm
* seq24_idx  the same with idx and FE
* plain      12 steps, no idx, no FE (left-padded input)
The graph constructor's parameters are drawn small (N(0, 0.05)), so tanh does not saturate and every row of the learned graph has a
clear gap between its k-th and (k+1)-th values; the make script checks that gap (2^-20 relative) at every forward."""
import gzip
import io
import math
import os

import torch

from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the tests)

FIXTURE = "mtgnn.pt.gz"

_BASE = dict(gcn_true=True, build_adj=True, gcn_depth=2, num_nodes=207, kernel_set=[2, 3, 6, 7], kernel_size=7, dropout=0.0,
             subgraph_size=20, node_dim=40, dilation_exponential=1, conv_channels=32, residual_channels=32, skip_channels=64,
             end_channels=128, seq_length=12, in_dim=2, out_dim=10, layers=3, propalpha=0.05, tanhalpha=3, layer_norm_affline=True,
             xd=None)
CASES = {
    "idx": dict(model=dict(_BASE), B=4, idx=True, fe=False, adj=False, seed=701),
    "fe": dict(model=dict(_BASE, xd=8), B=4, idx=False, fe=True, adj=False, seed=712),
    "predef": dict(model=dict(_BASE, build_adj=False), B=4, idx=False, fe=False, adj=True, seed=703),
    "nogcn_dil2": dict(model=dict(_BASE, gcn_true=False, dilation_exponential=2, layer_norm_affline=False), B=4, idx=False, fe=False,
                       adj=True, seed=704),
    "seq24": dict(model=dict(_BASE, seq_length=24, out_dim=5, layer_norm_affline=False), B=4, idx=False, fe=False, adj=False,
                  seed=705),
    "seq24_idx": dict(model=dict(_BASE, seq_length=24, out_dim=5, layer_norm_affline=False, xd=8), B=4, idx=True, fe=True, adj=False,
                      seed=716),
    "plain": dict(model=dict(_BASE), B=4, idx=False, fe=False, adj=False, seed=707),
}
STEPS, LR = 2, 1e-4


def build(cls, c):
    return cls(**c["model"])


def seeded_state(c, cls):
    """The parameters of case c from its seed (float32 values), in sorted key order: the graph constructor's N(0, 0.05), conv and linear
    weights N(0, 2 / (in + out)), LayerNorm weights 1 + N(0, 0.1), every other parameter N(0, 0.1)."""
    m = build(cls, c)
    g = torch.Generator().manual_seed(c["seed"])
    state = dict(m.state_dict())
    for k in sorted(dict(m.named_parameters())):
        shape = state[k].shape
        v = torch.randn(shape, generator=g, dtype=torch.float64)
        if k.startswith("_graph_constructor."):
            v = 0.05 * v
        elif k.endswith("_normalization._weight"):
            v = 1 + 0.1 * v
        elif k.endswith("weight") and len(shape) == 4:
            v = v * math.sqrt(2.0 / (shape[0] * shape[3] + shape[1] * shape[3]))
        else:
            v = 0.1 * v
        state[k] = v.float()
    return state


def adjacency(c):
    """A predefined graph: about ten random out-edges per node, weight 1, duplicates merged, no self loops."""
    n = c["model"]["num_nodes"]
    g = torch.Generator().manual_seed(c["seed"] + 1)
    A = torch.zeros(n, n)
    src = torch.arange(n).repeat_interleave(10)
    dst = torch.randint(0, n, (n * 10,), generator=g)
    A[src, dst] = 1.0
    A.fill_diagonal_(0.0)
    return A


def inputs(c, step):
    """(X (B, in_dim, N, seq), target (B, out_dim, N, 1)) of step `step`, float32: X uniform in [-1, 1), target N(0, 1)."""
    m = c["model"]
    g = torch.Generator().manual_seed(c["seed"] * 10 + step)
    X = 2 * torch.rand(c["B"], m["in_dim"], m["num_nodes"], m["seq_length"], generator=g) - 1
    Y = torch.randn(c["B"], m["out_dim"], m["num_nodes"], 1, generator=g)
    return X, Y


def extras(c):
    """(idx, FE, A_tilde) of case c, float32 / int64 on the CPU (None where the case has none)."""
    n = c["model"]["num_nodes"]
    g = torch.Generator().manual_seed(c["seed"] + 2)
    idx = torch.randperm(n, generator=g) if c["idx"] else None
    FE = torch.rand(n, c["model"]["xd"], generator=g) if c["fe"] else None
    A = adjacency(c) if c["adj"] else None
    return idx, FE, A


def model_for(c, cls, device, dtype):
    m = build(cls, c)
    m.load_state_dict(seeded_state(c, cls))
    return m.to(device=device, dtype=dtype)


def run(m, c, device, dtype, on_graph=None):
    """The case's training steps and eval call on model m -> {name: tensor}: out.<step>, loss.<step>, grad.<param>.<step>, out.eval.
    With `on_graph`, on_graph(graph_constructor, idx, FE) is called at every build of the learned graph."""
    idx, FE, A = extras(c)
    to = dict(device=device, dtype=dtype)
    idx = None if idx is None else idx.to(device)
    FE = None if FE is None else FE.to(**to)
    A = None if A is None else A.to(**to)
    hook = None
    if on_graph is not None:
        hook = m._graph_constructor.register_forward_pre_hook(
            lambda mod, args, kwargs: on_graph(mod, args[0], kwargs.get("FE", args[1] if len(args) > 1 else None)), with_kwargs=True)
    opt = torch.optim.Adam(m.parameters(), lr=LR)
    got = {}
    m.train()
    for s in range(STEPS):
        X, Y = inputs(c, s)
        X = X.to(**to)
        if idx is not None:
            X = X[:, :, idx, :]
        opt.zero_grad()
        out = m(X, A, idx=idx, FE=FE)
        loss = (out - Y.to(**to)).abs().mean()
        loss.backward()
        got[f"out.{s}"], got[f"loss.{s}"] = out.detach(), loss.detach().view(1)
        for k, p in m.named_parameters():
            got[f"grad.{k}.{s}"] = p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)
        opt.step()
    m.eval()
    X, _ = inputs(c, 99)
    X = X.to(**to)
    if idx is not None:
        X = X[:, :, idx, :]
    with torch.no_grad():
        got["out.eval"] = m(X, A, idx=idx, FE=FE)
    m.train()
    if hook is not None:
        hook.remove()
    return got


def reference_module():
    """The unmodified reference nn/attention/mtgnn.py."""
    from oracle import refload
    return refload.load("nn.attention.mtgnn")


def load(golden_dir):
    """The goldens (tests/golden/make_goldens_mtgnn.py), each case's stacked fingerprints unpacked into {key: fingerprint}."""
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        g = torch.load(io.BytesIO(f.read()), weights_only=False)
    for c in g["cases"].values():
        c["fingerprints"] = dict(zip(c.pop("fingerprint_keys"), c["fingerprints"]))
    return g
