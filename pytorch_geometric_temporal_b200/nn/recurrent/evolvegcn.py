"""EvolveGCNO and EvolveGCNH -- drop-ins for torch_geometric_temporal/nn/recurrent/evolvegcno.py and evolvegcnh.py: the reference's
constructors, `initial_weight` (1, C, C) glorot, `recurrent_layer` a torch.nn.GRU(C, C), -H's `pooling_layer.select.weight` (1, C) (PyG 2.x
TopKPooling's layout), so the state_dict keys and a seeded initialisation equal the reference's.  `self.weight` is a plain attribute
holding the (1, C, C) weight of the last call; `reinitialize_weight()` or assigning None restarts from `initial_weight`, and assigning
`weight.detach()` cuts the autograd chain, which otherwise runs through the carried weight across calls.

One call is W_t = GRU(W_{t-1}, W_{t-1}) (-O) or GRU(X~, W_{t-1}) with X~ = TopKPooling(X) (-H), then out = Op (X W_t), Op = gcn_norm's
operator (normalize=True) or the raw edge weights without self loops (normalize=False).  For 2-D float32 X and weights with 1 <= C <= 32
and edge_weight None or a float32 (E,) vector that needs no gradient, it runs on the row-split kernels (stmp_evolvegcn_rows_*, DESIGN
§4s): one launch for -O, two for -H, with a hand-written backward.  Everything else -- float64, C > 32, a gradient into edge_weight, or
`fused_training = False` for a training call -- runs op for op on the GPU (the plan and ops.spmm in float32, index_add otherwise, and the
module's own GRU).  `cached` is stored and has no effect, as in the reference, whose cache is never filled."""
import math

import torch

from ... import _lib, ops
from ...plan import PlanCache, _require_cuda


def glorot(t: torch.Tensor):
    """PyG's glorot: U(-a, a), a = sqrt(6 / (fan_in + fan_out)) over the last two dimensions."""
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)


def gcn_norm(edge_index, edge_weight, num_nodes, improved=False, add_self_loops=True, dtype=None):
    """PyG's gcn_norm on tensors (the op-for-op route outside float32 or with a gradient into edge_weight): the non-loop edges, then one
    loop per node whose weight is the graph's own loop weight where it has one, else 1 (2 when improved); D^-1/2 A D^-1/2 by destination
    degree."""
    fill = 2.0 if improved else 1.0
    if edge_weight is None:
        edge_weight = torch.ones(edge_index.size(1), dtype=dtype, device=edge_index.device)
    if add_self_loops:
        mask = edge_index[0] != edge_index[1]
        loop = torch.arange(num_nodes, device=edge_index.device, dtype=edge_index.dtype)
        loop_w = edge_weight.new_full((num_nodes,), fill)
        inv = ~mask
        loop_w[edge_index[0][inv]] = edge_weight[inv]
        edge_index = torch.cat([edge_index[:, mask], torch.stack([loop, loop])], dim=1)
        edge_weight = torch.cat([edge_weight[mask], loop_w])
    row, col = edge_index[0], edge_index[1]
    deg = edge_weight.new_zeros(num_nodes).index_add(0, col, edge_weight)
    dis = deg.pow(-0.5)
    dis = dis.masked_fill(dis == float("inf"), 0)
    return edge_index, dis[row] * edge_weight * dis[col]


def topk_size(ratio: float, num_nodes: int, dtype) -> int:
    """The nodes PyG's topk keeps: int(ratio) when ratio >= 1, else ceil(float(ratio) * N) computed in the score's dtype; at most N."""
    if ratio >= 1:
        k = int(ratio)
    else:
        k = int(math.ceil(float((float(ratio) * torch.tensor([num_nodes], dtype=dtype)).ceil())))
    return min(k, num_nodes)


class SelectTopK(torch.nn.Module):
    """PyG 2.x SelectTopK's parameter: `weight` (1, C), drawn U(-1/sqrt(C), 1/sqrt(C)) by its constructor."""

    def __init__(self, in_channels: int, ratio):
        super().__init__()
        self.in_channels, self.ratio = in_channels, ratio
        self.weight = torch.nn.Parameter(torch.empty(1, in_channels))
        self.reset_parameters()

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.in_channels)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)


class TopKPooling(torch.nn.Module):
    """PyG 2.x TopKPooling(in_channels, ratio)'s parameters and draws: SelectTopK's constructor draws `select.weight`, then TopKPooling's
    reset_parameters draws it again."""

    def __init__(self, in_channels: int, ratio):
        super().__init__()
        self.in_channels, self.ratio = in_channels, ratio
        self.select = SelectTopK(in_channels, ratio)
        self.reset_parameters()

    def reset_parameters(self):
        self.select.reset_parameters()

    def forward(self, x):
        """(x[perm] * s[perm], perm), s = tanh((x p) / |p|), perm = the first topk_size nodes of a stable descending sort of s."""
        p = self.select.weight
        score = torch.tanh((x * p).sum(dim=-1) / p.norm(p=2, dim=-1))
        k = topk_size(self.ratio, x.size(0), score.dtype)
        perm = torch.sort(score, descending=True, stable=True).indices[:k]
        return x[perm] * score[perm].view(-1, 1), perm


class _EvolveGCN(torch.nn.Module):
    """The routing, plans and convolution shared by EvolveGCNO and EvolveGCNH."""

    def _init_common(self, in_channels, improved, cached, normalize, add_self_loops):
        self.in_channels = in_channels
        self.improved, self.cached, self.normalize, self.add_self_loops = improved, cached, normalize, add_self_loops
        self._plans = PlanCache()
        self.fused_training = True      # False: op-for-op autograd path for training calls (tests compare the two)

    def reset_parameters(self):
        glorot(self.initial_weight)

    def reinitialize_weight(self):
        self.weight = None

    def _plan(self, edge_index, edge_weight, num_nodes):
        """gcn_norm's operator (STMP_FLAVOR_GCN: improved and add_self_loops as its flags) or, with normalize=False, the raw edge weights
        (the add GatedGraphConv plan: no self loops, duplicates kept)."""
        if not self.normalize:
            return self._plans.get_gated(edge_index, edge_weight, num_nodes, "add")
        flags = (_lib.GCN_IMPROVED if self.improved else 0) | (0 if self.add_self_loops else _lib.GCN_NO_SELF_LOOPS)
        return self._plans.get(_lib.FLAVOR_GCN, edge_index, edge_weight, num_nodes, flags=flags)

    def _fused_ok(self, X, W_prev, edge_weight, training):
        """The module's conditions for the row-split kernels: 2-D float32 X of C in 1..32 channels on at least one node, float32 parameters
        and carried weight, edge_weight None or a float32 (E,) vector that needs no gradient; training calls also need `fused_training`."""
        C = self.in_channels
        if X.dim() != 2 or X.dtype != torch.float32 or X.size(1) != C or not 1 <= C <= 32 or X.size(0) < 1:
            return False
        if W_prev.dtype != torch.float32 or any(p.dtype != torch.float32 for p in self.parameters()):
            return False
        if edge_weight is not None and (edge_weight.dtype != torch.float32 or edge_weight.dim() != 1 or edge_weight.requires_grad):
            return False
        return not (training and not self.fused_training)

    def _conv(self, W, X, edge_index, edge_weight):
        """GCNConv_Fixed_W op for op: Op (X W)."""
        XW = torch.matmul(X, W)
        if XW.dtype == torch.float32 and (edge_weight is None or not edge_weight.requires_grad):
            return ops.spmm(self._plan(edge_index, edge_weight, X.size(0)), 0, XW)
        if self.normalize:
            edge_index, edge_weight = gcn_norm(edge_index, edge_weight, X.size(0), self.improved, self.add_self_loops, XW.dtype)
        msg = XW.index_select(0, edge_index[0])
        if edge_weight is not None:
            msg = edge_weight.view(-1, 1).to(XW.dtype) * msg
        return XW.new_zeros(XW.shape).index_add(0, edge_index[1], msg)

    def _step(self, X, edge_index, edge_weight, p):
        _require_cuda(X, "X")
        C = self.in_channels
        W_prev = self.initial_weight if self.weight is None else self.weight
        r = self.recurrent_layer
        params = list(self.parameters())
        needs_grad = torch.is_grad_enabled() and (any(q.requires_grad for q in params) or X.requires_grad or W_prev.requires_grad)
        if self._fused_ok(X, W_prev, edge_weight, needs_grad):
            plan = self._plan(edge_index, edge_weight, X.size(0))
            if ops.evolvegcn_rows_supported(plan, C):
                args = (plan, X, W_prev.reshape(C, C), r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0, p)
                if needs_grad:
                    out, W_new = ops.evolvegcn_rows_train(*args)
                else:
                    out, W_new = ops.evolvegcn_rows_fwd(*args)[:2]
                self.weight = W_new.unsqueeze(0)
                return out
        if p is None:
            _, self.weight = r(W_prev, W_prev)
        else:
            X_tilde = self.pooling_layer(X)[0]
            _, self.weight = r(X_tilde[None, :, :], W_prev)
        return self._conv(self.weight.squeeze(dim=0), X, edge_index, edge_weight)


class EvolveGCNO(_EvolveGCN):
    def __init__(self, in_channels: int, improved: bool = False, cached: bool = False, normalize: bool = True, add_self_loops: bool = True):
        super().__init__()
        self._init_common(in_channels, improved, cached, normalize, add_self_loops)
        self.initial_weight = torch.nn.Parameter(torch.empty(1, in_channels, in_channels))
        self.weight = None
        self.recurrent_layer = torch.nn.GRU(input_size=in_channels, hidden_size=in_channels, num_layers=1)
        self.reset_parameters()

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None) -> torch.FloatTensor:
        return self._step(X, edge_index, edge_weight, None)


class EvolveGCNH(_EvolveGCN):
    def __init__(self, num_of_nodes: int, in_channels: int, improved: bool = False, cached: bool = False, normalize: bool = True,
                 add_self_loops: bool = True):
        super().__init__()
        self._init_common(in_channels, improved, cached, normalize, add_self_loops)
        self.num_of_nodes = num_of_nodes
        self.weight = None
        self.initial_weight = torch.nn.Parameter(torch.empty(1, in_channels, in_channels))
        self.ratio = self.in_channels / self.num_of_nodes
        self.pooling_layer = TopKPooling(self.in_channels, self.ratio)
        self.recurrent_layer = torch.nn.GRU(input_size=in_channels, hidden_size=in_channels, num_layers=1)
        self.reset_parameters()

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None) -> torch.FloatTensor:
        k = topk_size(self.ratio, X.size(0), X.dtype)
        if k != self.in_channels:
            raise RuntimeError(f"EvolveGCNH: TopKPooling keeps {k} of {X.size(0)} nodes (ratio {self.ratio}), but the GRU's hidden state "
                               f"has batch {self.in_channels}: Expected hidden size (1, {k}, {self.in_channels}), got "
                               f"[1, {self.in_channels}, {self.in_channels}]")
        return self._step(X, edge_index, edge_weight, self.pooling_layer.select.weight.view(-1))
