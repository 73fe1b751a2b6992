"""HeteroGCLSTM -- drop-in for torch_geometric_temporal/nn/hetero/heterogclstm.py: constructor `(in_channels_dict, out_channels, metadata,
bias=True)`, `forward(x_dict, edge_index_dict, h_dict=None, c_dict=None) -> (h_dict, c_dict)`, the reference's attributes and state_dict
keys (`conv_i.convs.<src___rel___dst>.lin_l.weight`, ..., `W_i.<type>`, `b_i.<type>`, gate by gate) and its initialisation: glorot `W_*`
and `b_*` at construction, the SAGEConvs' lazy `lin_l` / `lin_r` materialised at the first forward in PyG's call order.

Per node type t and gate g: pre_g = X_t W_g + b_g + sum over the edge types e = (s, rel, t) of mean_e(H_s) lin_l^T + lin_l.bias + H_t lin_r^T
(PyG HeteroConv of SAGEConvs, aggr "sum"), then the LSTM without peepholes.  Inside the envelope every node type runs in one launch of
stmp_hetero_lstm_fwd (DESIGN §4v): float32 2-D X with in_channels <= 32 for every type, out 32 with at most four incoming edge types per
type or out 64 with one, at most eight node types.  A call that needs gradients (parameters or inputs requiring grad) trains on the same
launch with a stash, and its backward is stmp_hetero_lstm_bwd (at most four launches), when `fused_training` is set, every node type of
x_dict is an output and no type has more than eight outgoing edge types.  Everything else runs op for op on the GPU (the float32
means through spmm on the bipartite plans, float64 by index_add, torch matmuls, autograd).

The one deliberate deviation: with h_dict / c_dict None the reference builds CPU zeros in the default dtype, so it cannot run on GPU
inputs; here the zeros are made on X's device in X's dtype."""
import math

import torch
from torch.nn import Parameter, UninitializedParameter
from torch.nn.parameter import is_lazy

from ... import _lib, ops
from ...plan import PlanCache, _require_cuda
from ..recurrent._cheb import glorot_

GATES = "ifco"


def conv_key(edge_type) -> str:
    """PyG ModuleDict's key of an edge-type tuple, `<src___rel___dst>` (older PyG releases used `src__rel__dst`)."""
    return "<" + "___".join(edge_type) + ">"


class LazyLinear(torch.nn.Module):
    """PyG `Linear(-1, out, bias)`: `weight` is an UninitializedParameter until `materialize(in_channels)` (or a state_dict load) gives it
    its shape; PyG's default initialisation, kaiming-uniform with fan = in and a = sqrt(5) for the weight, then uniform with bound
    1 / sqrt(in) for the bias, drawn on the parameters' device."""

    def __init__(self, out_channels: int, bias: bool):
        super().__init__()
        self.in_channels, self.out_channels = -1, out_channels
        self.weight = UninitializedParameter()
        if bias:
            self.bias = Parameter(torch.empty(out_channels))
        else:
            self.register_parameter("bias", None)
        self._register_load_state_dict_pre_hook(self._lazy_load_hook)

    def materialize(self, in_channels: int):
        self.in_channels = in_channels
        self.weight.materialize((self.out_channels, in_channels))
        with torch.no_grad():
            bound = math.sqrt(6 / ((1 + math.sqrt(5) ** 2) * in_channels))
            self.weight.uniform_(-bound, bound)
            if self.bias is not None:
                bound = 1.0 / math.sqrt(in_channels)
                self.bias.uniform_(-bound, bound)

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        # an uninitialised weight is saved as it is (detaching it raises), as PyG's Linear does
        for name, v in (("weight", self.weight), ("bias", self.bias)):
            if v is not None:
                destination[prefix + name] = v if keep_vars or is_lazy(v) else v.detach()

    def _lazy_load_hook(self, state_dict, prefix, *args):
        w = state_dict.get(prefix + "weight")
        if w is not None and is_lazy(self.weight) and not is_lazy(w):
            self.in_channels = w.size(-1)
            self.weight.materialize(w.shape)


class SAGEParams(torch.nn.Module):
    """PyG `SAGEConv((-1, -1), out, bias=bias)`'s parameters: `lin_l` (with bias) on the mean of the sources, `lin_r` (no bias) on the
    destination's own row."""

    def __init__(self, out_channels: int, bias: bool):
        super().__init__()
        self.in_channels, self.out_channels, self.aggr = (-1, -1), out_channels, "mean"
        self.lin_l = LazyLinear(out_channels, bias)
        self.lin_r = LazyLinear(out_channels, False)


class HeteroConvParams(torch.nn.Module):
    """PyG `HeteroConv({edge_type: SAGEConv}, aggr="sum")`'s parameters: `convs`, keyed by `conv_key`, in metadata order."""

    def __init__(self, edge_types, out_channels: int, bias: bool):
        super().__init__()
        self.aggr = "sum"
        self.edge_types = [tuple(e) for e in edge_types]
        self.convs = torch.nn.ModuleDict({conv_key(e): SAGEParams(out_channels, bias) for e in self.edge_types})

    def conv(self, edge_type) -> SAGEParams:
        return self.convs[conv_key(edge_type)]


class HeteroGCLSTM(torch.nn.Module):
    def __init__(self, in_channels_dict: dict, out_channels: int, metadata: tuple, bias: bool = True):
        super().__init__()
        self.in_channels_dict, self.out_channels, self.metadata, self.bias = in_channels_dict, out_channels, metadata, bias
        # registration order mirrors the reference (conv, W, b per gate), so the state_dict keys come in its order
        for g in GATES:
            setattr(self, f"conv_{g}", HeteroConvParams(metadata[1], out_channels, bias))
            setattr(self, f"W_{g}", torch.nn.ParameterDict({t: Parameter(torch.empty(c, out_channels)) for t, c in in_channels_dict.items()}))
            setattr(self, f"b_{g}", torch.nn.ParameterDict({t: Parameter(torch.empty(1, out_channels)) for t in in_channels_dict}))
        for p in ("W", "b"):                  # the reference's _set_parameters: every W_* (gate order), then every b_*
            for g in GATES:
                for t in in_channels_dict:
                    glorot_(getattr(self, f"{p}_{g}")[t])
        self._plans = PlanCache(max_entries=4 * max(1, len(metadata[1])))
        self._packs = {}
        self.fused_training = True      # False: op-for-op autograd path for training calls (tests compare the two)

    # ---- structure of one call ---------------------------------------------------------------------------------------------------
    def _edges(self, edge_index_dict):
        """The edge types HeteroConv runs: metadata order, present in edge_index_dict (others are skipped or ignored)."""
        return [e for e in self.conv_i.edge_types if e in edge_index_dict]

    def materialize(self, edges):
        """The lazy lin_l / lin_r of `edges` that are still uninitialised, in the reference's first-forward order: gates i, f, c, o, edge
        types in metadata order, lin_l (weight, bias) before lin_r.  Both read states of out_channels columns."""
        for g in GATES:
            hc = getattr(self, f"conv_{g}")
            for e in edges:
                conv = hc.conv(e)
                for lin in (conv.lin_l, conv.lin_r):
                    if is_lazy(lin.weight):
                        lin.materialize(self.out_channels)

    def _check(self, x_dict, edge_index_dict, h_dict, c_dict):
        """(output types, edges, incoming edges per output type); raises the reference's KeyErrors and every shape error before a launch."""
        for t, X in x_dict.items():
            if t not in self.W_i:
                raise KeyError(t)
            if X.size(-1) != self.W_i[t].size(0):
                raise RuntimeError(f"x_dict[{t!r}] has {X.size(-1)} channels, in_channels_dict gives {self.W_i[t].size(0)}")
        edges = self._edges(edge_index_dict)
        for e in edges:
            for t in (e[0], e[2]):
                if t not in x_dict:
                    raise KeyError(t)
        out_types = list(c_dict) if c_dict is not None else list(x_dict)
        incoming = {t: [e for e in edges if e[2] == t] for t in out_types}
        for t in out_types:
            if t not in x_dict or not incoming[t]:       # the reference: conv_i[node_type] has no entry for a type without in-edges
                raise KeyError(t)
        for name, d in (("h_dict", h_dict), ("c_dict", c_dict)):
            for t, S in (d or {}).items():
                if t in x_dict and S.shape[-2:] != (x_dict[t].size(-2), self.out_channels):
                    raise RuntimeError(f"{name}[{t!r}] has shape {tuple(S.shape)}, want ({x_dict[t].size(-2)}, {self.out_channels})")
        for t, X in x_dict.items():
            _require_cuda(X, f"x_dict[{t!r}]")
        return out_types, edges, incoming

    def _plan(self, edge_index_dict, x_dict, e):
        return self._plans.get_bipartite(edge_index_dict[e], x_dict[e[0]].size(-2), x_dict[e[2]].size(-2))

    # ---- fused route ---------------------------------------------------------------------------------------------------------------
    def _fused_ok(self, x_dict, h_dict, c_dict, out_types, incoming, training):
        """The one-launch route: see the module docstring.  Training also needs `fused_training`, every node type of x_dict among the
        outputs (each source's state gradient is gathered in the same table) and at most eight outgoing edge types per node type."""
        if len(out_types) > _lib.HETERO_MAX_TYPES:
            return False
        if training:
            if not self.fused_training or set(out_types) != set(x_dict):
                return False
            outgoing = [e[0] for t in out_types for e in incoming[t]]
            if any(outgoing.count(s) > 8 for s in set(outgoing)):
                return False
        for t in out_types:
            X = x_dict[t]
            if X.dim() != 2 or X.dtype != torch.float32 or X.size(0) < 1:
                return False
            if not ops.hetero_lstm_supported(self.out_channels, X.size(1), len(incoming[t])):
                return False
        for d in (h_dict, c_dict):
            if d is not None and any(S.dtype != torch.float32 or S.dim() != 2 for S in d.values()):
                return False
        return True

    def _spec(self, t, edges):
        """(params, spec) of type t: every parameter its packed weight is made of and the block of the packed weight / bias gradient it
        receives (ops._spec_grads).  Every lin_r^e into t receives the same root block, every lin_l^e.bias the summed bias's gradient."""
        params, spec = [], []
        Co, Ci = self.out_channels, self.W_i[t].size(0)
        for gi, g in enumerate(GATES):
            row = gi * Co
            params += [getattr(self, f"W_{g}")[t], getattr(self, f"b_{g}")[t]]
            spec += [("wt", row, Co, 0, Ci), ("b", row, Co)]
            for r, e in enumerate(edges):
                conv = getattr(self, f"conv_{g}").conv(e)
                params += [conv.lin_l.weight, conv.lin_r.weight]
                spec += [("w", row, Co, Ci + Co * (1 + r), Co), ("w", row, Co, Ci, Co)]
                if self.bias:
                    params.append(conv.lin_l.bias)
                    spec.append(("b", row, Co))
        return params, spec

    def _packed(self, t, edges):
        """(w (4 out, nb), b (4 out)) of type t: per gate [W_g^T | sum_e lin_r^e | lin_l^{e_1} | ...], b_g + sum_e lin_l^e.bias, summed
        in edge-type order; rebuilt when a parameter changes."""
        params = self._spec(t, edges)[0]

        def build():
            ws, bs = [], []
            for g in GATES:
                convs = [getattr(self, f"conv_{g}").conv(e) for e in edges]
                root = convs[0].lin_r.weight
                for c in convs[1:]:
                    root = root + c.lin_r.weight
                ws.append(torch.cat([getattr(self, f"W_{g}")[t].t(), root] + [c.lin_l.weight for c in convs], dim=1))
                b = getattr(self, f"b_{g}")[t].reshape(-1)
                if self.bias:
                    for c in convs:
                        b = b + c.lin_l.bias
                bs.append(b)
            return torch.cat(ws).float().contiguous(), torch.cat(bs).float().contiguous()
        cache = self._packs.setdefault((t, tuple(edges)), ops.PackCache())
        return cache.get(params, build)

    def _fused(self, x_dict, edge_index_dict, h_dict, c_dict, out_types, incoming, edges, training):
        types, params, specs = [], [], []
        for t in out_types:
            w, b = self._packed(t, incoming[t])
            plans = [self._plan(edge_index_dict, x_dict, e) for e in incoming[t]]
            sources = [None if h_dict is None else h_dict[e[0]] for e in incoming[t]]
            src_idx = [out_types.index(e[0]) if e[0] in out_types else -1 for e in incoming[t]]
            ranks = [edges.index(e) for e in incoming[t]]
            types.append((x_dict[t], None if h_dict is None else h_dict[t], None if c_dict is None else c_dict[t], w, b, plans, sources,
                          src_idx, ranks))
            if training:
                p, sp = self._spec(t, incoming[t])
                params += p
                specs.append(sp)
        if training:
            outs = ops.hetero_lstm_train(self.out_channels, types, params, specs)
        else:
            outs = ops.hetero_lstm_fwd(self.out_channels, types, h_dict is not None)
        return {t: o[0] for t, o in zip(out_types, outs)}, {t: o[1] for t, o in zip(out_types, outs)}

    # ---- op for op -------------------------------------------------------------------------------------------------------------------
    def _gate(self, g, t, x_dict, edge_index_dict, h_dict, incoming):
        hc = getattr(self, f"conv_{g}")
        conv_sum = None
        for e in incoming[t]:
            c = hc.conv(e)
            mean = ops.bipartite_mean(self._plan(edge_index_dict, x_dict, e), edge_index_dict[e], h_dict[e[0]])
            out = torch.nn.functional.linear(mean, c.lin_l.weight, c.lin_l.bias) + torch.nn.functional.linear(h_dict[t], c.lin_r.weight)
            conv_sum = out if conv_sum is None else conv_sum + out
        return torch.matmul(x_dict[t], getattr(self, f"W_{g}")[t]) + conv_sum + getattr(self, f"b_{g}")[t]

    def forward(self, x_dict, edge_index_dict, h_dict=None, c_dict=None):
        out_types, edges, incoming = self._check(x_dict, edge_index_dict, h_dict, c_dict)
        self.materialize(edges)
        training = torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters())
                                                or any(v.requires_grad for d in (x_dict, h_dict, c_dict) if d for v in d.values()))
        if self._fused_ok(x_dict, h_dict, c_dict, out_types, incoming, training):
            return self._fused(x_dict, edge_index_dict, h_dict, c_dict, out_types, incoming, edges, training)
        zeros = lambda X: torch.zeros(X.size(-2), self.out_channels, device=X.device, dtype=X.dtype)
        if h_dict is None:
            h_dict = {t: zeros(X) for t, X in x_dict.items()}
        if c_dict is None:
            c_dict = {t: zeros(X) for t, X in x_dict.items()}
        h_out, c_out = {}, {}
        for t in out_types:
            pre = {g: self._gate(g, t, x_dict, edge_index_dict, h_dict, incoming) for g in GATES}
            C = torch.sigmoid(pre["f"]) * c_dict[t] + torch.sigmoid(pre["i"]) * torch.tanh(pre["c"])
            c_out[t] = C
            h_out[t] = torch.sigmoid(pre["o"]) * torch.tanh(C)   # no peephole: O does not read the new cell state
        return h_out, c_out
