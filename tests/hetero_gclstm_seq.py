"""HeteroGCLSTM cases shared by tests/golden/make_goldens_hetero_gclstm.py and the CPU / GPU HeteroGCLSTM tests.

It holds the float64 oracle's PyG layers.  PyG is not a dependency, so `Linear` (lazy, in_channels = -1), `SAGEConv` and `HeteroConv`
restate PyG's documented behaviour, the way tests/lrgcn_seq.py restates RGCNConv; `install()` puts them into the oracle/stubs
`torch_geometric.nn` namespace so the unmodified reference heterogclstm.py can run on them.  Version-sensitive choices (DESIGN §4v):
HeteroConv runs its convs in their (metadata) order and sums them by stacking; ModuleDict keys are `<src___rel___dst>`; lazy Linear
materialises at its first call with kaiming-uniform (fan = in, a = sqrt(5)) then a uniform bias of bound 1 / sqrt(in).

Cases: `unit` is the reference's unit-test shape (50 authors with 20 features, 50 papers with 30, out 32, `writes` plus ToUndirected's
`rev_writes`), two calls, H None then carried; `three32` / `three64` are three-type sequences of T snapshots through
StaticHeteroGraphTemporalSignal with unequal node counts, a self-relation, a type with several incoming edge types (out 32 only),
duplicate edges, isolated destinations and an E = 0 edge type, H / C carried from leaf H0 / C0, a per-type Linear head and a cumulative
MSE.  Graphs, features and parameters all come from the case's seeds."""
import gzip
import io
import math
import os

import torch

from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the goldens and tests)

FIXTURE = "hetero_gclstm.pt.gz"


# ---- restated PyG layers ------------------------------------------------------------------------------------------------------------
class Linear(torch.nn.Module):
    def __init__(self, in_channels, out_channels, bias=True):
        super().__init__()
        assert in_channels == -1
        self.in_channels, self.out_channels = in_channels, out_channels
        self.weight = torch.nn.parameter.UninitializedParameter()
        if bias:
            self.bias = torch.nn.Parameter(torch.empty(out_channels))
        else:
            self.register_parameter("bias", None)

    def forward(self, x):
        if isinstance(self.weight, torch.nn.parameter.UninitializedParameter):
            self.in_channels = x.size(-1)
            self.weight.materialize((self.out_channels, self.in_channels))
            a = math.sqrt(5)
            bound = math.sqrt(6 / ((1 + a ** 2) * self.in_channels))
            self.weight.data.uniform_(-bound, bound)
            if self.bias is not None:
                bound = 1.0 / math.sqrt(self.in_channels)
                self.bias.data.uniform_(-bound, bound)
        return torch.nn.functional.linear(x, self.weight, self.bias)

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        # an uninitialised weight is saved as it is (detaching it raises), as PyG's Linear does
        for name, v in (("weight", self.weight), ("bias", self.bias)):
            if v is not None:
                destination[prefix + name] = v if keep_vars or isinstance(v, torch.nn.parameter.UninitializedParameter) else v.detach()


class SAGEConv(torch.nn.Module):
    """SAGEConv(in, out, bias) with aggr "mean", root weight, no normalisation: lin_l(mean_j x_j) + lin_r(x_i)."""

    def __init__(self, in_channels, out_channels, bias=True):
        super().__init__()
        self.lin_l = Linear(-1, out_channels, bias=bias)
        self.lin_r = Linear(-1, out_channels, bias=False)

    def forward(self, x, edge_index):
        xs, xd = (x, x) if torch.is_tensor(x) else x
        src, dst = edge_index[0], edge_index[1]
        agg = torch.zeros(xd.size(0), xs.size(1), dtype=xs.dtype).index_add_(0, dst, xs[src])
        cnt = torch.zeros(xd.size(0), dtype=xs.dtype).index_add_(0, dst, torch.ones(dst.numel(), dtype=xs.dtype))
        out = self.lin_l(agg / cnt.clamp(min=1).unsqueeze(1))
        return out + self.lin_r(xd)


class _ModuleDict(torch.nn.ModuleDict):
    def __init__(self, d):
        super().__init__({"<" + "___".join(k) + ">": v for k, v in d.items()})

    def items_typed(self):
        return [(tuple(k[1:-1].split("___")), v) for k, v in self.items()]


class HeteroConv(torch.nn.Module):
    def __init__(self, convs, aggr="sum"):
        super().__init__()
        self.convs, self.aggr = _ModuleDict(convs), aggr

    def forward(self, x_dict, edge_index_dict):
        out = {}
        for edge_type, conv in self.convs.items_typed():
            if edge_type not in edge_index_dict:
                continue
            src, _, dst = edge_type
            x = x_dict[src] if src == dst else (x_dict.get(src), x_dict.get(dst))
            out.setdefault(dst, []).append(conv(x, edge_index_dict[edge_type]))
        return {k: torch.stack(v, 0).sum(0) for k, v in out.items()}


def install():
    """Makes the restated layers importable as torch_geometric.nn.SAGEConv / HeteroConv from the oracle stubs."""
    import sys
    from oracle import refload
    if refload._STUBS not in sys.path:
        sys.path.insert(0, refload._STUBS)
    import torch_geometric.nn as tgnn
    tgnn.SAGEConv, tgnn.HeteroConv = SAGEConv, HeteroConv


def reference_class():
    install()
    from oracle import refload
    return refload.load("nn.hetero.heterogclstm").HeteroGCLSTM


# ---- cases ------------------------------------------------------------------------------------------------------------------------
def _edges(g, n_src, n_dst, count):
    return torch.stack([torch.randint(0, n_src, (count,), generator=g), torch.randint(0, n_dst, (count,), generator=g)])


def unit_graph(seed=0):
    g = torch.Generator().manual_seed(seed)
    n = 50
    keep = torch.rand(n, n, generator=g, dtype=torch.float64) < 0.1
    writes = keep.triu(1).nonzero().t().contiguous()
    x = {"author": torch.rand(n, 20, generator=g, dtype=torch.float64), "paper": torch.rand(n, 30, generator=g, dtype=torch.float64)}
    ei = {("author", "writes", "paper"): writes, ("paper", "rev_writes", "author"): writes.flip(0).contiguous()}
    metadata = (["author", "paper"], list(ei))
    return x, ei, metadata, {"author": 20, "paper": 30}


def three_graph(out, seed=1, T=8):
    """(feature dicts, edge_index_dict (numpy), metadata, in_channels_dict): types a (37 nodes), b (50), c (9)."""
    g = torch.Generator().manual_seed(seed)
    n = {"a": 37, "b": 50, "c": 9}
    cin = {"a": 5, "b": 12, "c": 3}
    ab = _edges(g, 37, 40, 120)                       # b rows 40..49 are isolated
    ab = torch.cat([ab, ab[:, :15]], 1)               # duplicates
    ei = {("a", "to", "b"): ab, ("b", "rev", "a"): _edges(g, 50, 30, 90), ("a", "to", "c"): torch.zeros(2, 0, dtype=torch.int64)}
    if out == 32:                                     # b: three incoming edge types, one a self-relation
        ei[("b", "self", "b")] = _edges(g, 50, 50, 70)
        ei[("c", "to", "b")] = _edges(g, 9, 50, 20)
    feats = [{t: torch.randn(n[t], cin[t], generator=g, dtype=torch.float64).numpy() for t in n} for _ in range(T)]
    targets = [{t: torch.randn(n[t], generator=g, dtype=torch.float64).numpy() for t in n} for _ in range(T)]
    metadata = (list(n), list(ei))
    return feats, targets, {k: v.numpy() for k, v in ei.items()}, metadata, cin


CASES = {"unit": dict(kind="unit", out=32, seed=10), "three32": dict(kind="three", out=32, seed=11), "three64": dict(kind="three", out=64, seed=12)}


def build(cls, case, device="cpu", dtype=torch.float64):
    """(model, inputs) of a case; the model's parameters come from the case's seed, drawn on the CPU: construction, then the lazy
    materialisation in the reference's first-forward order (the reference materialises in its first call; the module through
    `materialize`, so both draw the same numbers)."""
    if case["kind"] == "unit":
        x, ei, metadata, cin = unit_graph()
        inputs = dict(x=x, ei=ei)
    else:
        feats, targets, ei_np, metadata, cin = three_graph(case["out"])
        inputs = dict(feats=feats, targets=targets, ei_np=ei_np)
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)            # the goldens' parameters are float64 draws
    try:
        torch.manual_seed(case["seed"])
        m = cls(in_channels_dict=cin, out_channels=case["out"], metadata=metadata)
        if hasattr(m, "materialize"):
            m.materialize([tuple(e) for e in metadata[1]])
    finally:
        torch.set_default_dtype(default)
    return m.to(device, dtype), inputs, metadata, cin


def materialize_reference(m, inputs, metadata):
    """Runs the reference once on zeros so its lazy layers draw their parameters (a forward consumes no other random numbers)."""
    if "x" in inputs:
        x, ei = inputs["x"], inputs["ei"]
    else:
        x = {t: torch.zeros(v.shape, dtype=torch.float64) for t, v in inputs["feats"][0].items()}
        ei = {k: torch.as_tensor(v) for k, v in inputs["ei_np"].items()}
    m(x, ei)


def run(m, case, inputs, metadata, device, dtype, signal_cls=None, grad=True):
    """Runs a case; returns (outputs dict, grads dict).  Gradients are of the sum of every output for `unit`, of the cumulative MSE of a
    per-type Linear head (seeded) for `three*`, with respect to X (unit) or H0 / C0 (three*) and every parameter."""
    outs = {}
    if case["kind"] == "unit":
        x = {t: v.to(device, dtype).requires_grad_(grad) for t, v in inputs["x"].items()}
        ei = {k: v.to(device) for k, v in inputs["ei"].items()}
        h, c = m(x, ei)
        h2, c2 = m(x, ei, h, c)
        loss = 0
        for k, d in (("h1", h), ("c1", c), ("h2", h2), ("c2", c2)):
            for t, v in d.items():
                outs[f"{k}.{t}"] = v
                loss = loss + v.sum() * (1.0 + 0.1 * len(t))
        leaves = {f"x.{t}": v for t, v in x.items()}
    else:
        sig = signal_cls(inputs["ei_np"], None, inputs["feats"], inputs["targets"])
        g = torch.Generator().manual_seed(case["seed"] + 100)
        types = metadata[0]
        heads = {t: (torch.randn(case["out"], generator=g, dtype=torch.float64).to(device, dtype),) for t in types}
        h0 = {t: (0.1 * torch.randn(v.shape[0], case["out"], generator=g, dtype=torch.float64)).to(device, dtype).requires_grad_(grad)
              for t, v in inputs["feats"][0].items()}
        c0 = {t: (0.1 * torch.randn(v.shape[0], case["out"], generator=g, dtype=torch.float64)).to(device, dtype).requires_grad_(grad)
              for t, v in inputs["feats"][0].items()}
        h, c = h0, c0
        loss = 0
        for step, snap in enumerate(sig):
            snap = snap.to(device) if hasattr(snap, "to") and device != "cpu" else snap
            xd = {t: v.to(device, dtype) for t, v in snap.x_dict.items()}
            h, c = m(xd, snap.edge_index_dict, h, c)
            for t in types:
                pred = h[t] @ heads[t][0]
                loss = loss + ((pred - snap[t].y.to(device, dtype)) ** 2).mean()
                outs[f"h{step}.{t}"] = h[t]
            for t in types:
                outs[f"c{step}.{t}"] = c[t]
        loss = loss / sig.snapshot_count
        leaves = {**{f"h0.{t}": v for t, v in h0.items()}, **{f"c0.{t}": v for t, v in c0.items()}}
    if not grad:
        return {k: v.detach() for k, v in outs.items()}, {}, loss.detach()
    params = dict(m.named_parameters())
    grads = torch.autograd.grad(loss, list(leaves.values()) + list(params.values()), allow_unused=True)
    names = list(leaves) + [f"p.{k}" for k in params]
    gd = {k: (torch.zeros_like(v) if gr is None else gr) for k, v, gr in zip(names, list(leaves.values()) + list(params.values()), grads)}
    return {k: v.detach() for k, v in outs.items()}, {k: v.detach() for k, v in gd.items()}, loss.detach()


def load(golden_dir):
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)["cases"]


def fingerprint_close(got, want, rtol):
    """A fingerprint within rtol of the reference's norm in each projection and in the norm."""
    return bool(((fingerprint(got) - want).abs() <= rtol * want[-1].abs() + 1e-12).all())
