"""LRGCN -- drop-in for torch_geometric_temporal/nn/recurrent/lrgcn.py: constructor `(in_channels, out_channels, num_relations,
num_bases)`, `forward(X, edge_index, edge_type, H=None, C=None) -> (H, C)`, eight PyG RGCNConvs `conv_{x,h}_{i,f,c,o}` with the state_dict
keys `weight`, `comp` (absent when num_bases is None), `root`, `bias` in that order and PyG's initialisation order (glorot weight, comp,
root; zero bias), so a seeded model equals the reference's.

A gate is RGCNConv(X) + RGCNConv(H), and an RGCNConv is a root product plus one mean-aggregated hop per relation, so one LRGCN step is the
graph-LSTM cell without peepholes on the basis [X | H | Op_0 X | Op_0 H | ...] with one operator per relation: the row-split LSTM cell
(stmp_lstm_rows_*) serves it for in_channels <= 16 at 32 channels with one or two relations and at 64 channels with one, one launch per
step for inference and training alike (DESIGN §4q).  Everything else -- more relations, other widths, wider inputs, batched X, or
`fused_training = False` for a training call -- runs op for op on the GPU (ops.spmm per relation, torch matmuls, autograd)."""
import torch

from ... import _lib, ops
from ...plan import RgcnPlan, _require_cuda
from ._cheb import glorot_


class RGCNParams(torch.nn.Module):
    """Parameter holder with PyG RGCNConv's state_dict layout: `weight` (B, in, out) and `comp` (R, B) with bases, else `weight` (R, in,
    out); `root` (in, out); `bias` (out)."""

    def __init__(self, in_channels, out_channels, num_relations, num_bases):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.num_relations, self.num_bases = num_relations, num_bases
        P = torch.nn.Parameter
        if num_bases is not None:
            self.weight = P(torch.empty(num_bases, in_channels, out_channels))
            self.comp = P(torch.empty(num_relations, num_bases))
        else:
            self.weight = P(torch.empty(num_relations, in_channels, out_channels))
            self.register_parameter("comp", None)
        self.root = P(torch.empty(in_channels, out_channels))
        self.bias = P(torch.empty(out_channels))
        glorot_(self.weight)
        if self.comp is not None:
            glorot_(self.comp)
        glorot_(self.root)
        torch.nn.init.zeros_(self.bias)

    def relation_weights(self) -> torch.Tensor:
        """W (R, in, out): W_r = sum_b comp[r, b] V_b with bases, else the weight itself."""
        if self.comp is None:
            return self.weight
        return (self.comp @ self.weight.view(self.num_bases, -1)).view(self.num_relations, self.in_channels, self.out_channels)


def relation_ids(edge_type: torch.Tensor, num_relations: int) -> torch.Tensor:
    """int64 relation of every edge, -1 for none, on the device and without a host sync: the relation r with `edge_type == r` (the
    reference's per-relation mask), so an integer-valued float selects its relation and any other float (non-integral, inf, NaN) or a
    value outside [0, num_relations) selects none."""
    t = edge_type.detach().reshape(-1)
    if t.is_floating_point():
        ok = torch.isfinite(t) & (t == torch.floor(t)) & (t >= 0) & (t < num_relations)
    else:
        ok = (t >= 0) & (t < num_relations)
    return torch.where(ok, t, torch.zeros_like(t)).to(torch.int64).masked_fill_(~ok, -1)


class LRGCN(torch.nn.Module):
    def __init__(self, in_channels: int, out_channels: int, num_relations: int, num_bases: int):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.num_relations, self.num_bases = num_relations, num_bases
        # creation order mirrors the reference (lrgcn.py, _create_layers), so seeded init consumes the RNG identically
        for g in "ifco":
            setattr(self, f"conv_x_{g}", RGCNParams(in_channels, out_channels, num_relations, num_bases))
            setattr(self, f"conv_h_{g}", RGCNParams(out_channels, out_channels, num_relations, num_bases))
        self._plans = {}
        self._rows_pack = ops.PackCache()
        self.fused_training = True      # False: op-for-op autograd path for training calls (tests compare the two)

    def _relation_plans(self, edge_index, edge_type, num_nodes):
        """ceil(R / 2) plans of two relations each (the last may hold one), cached on (data_ptr, _version, shape) of edge_index and
        edge_type: no device sync on a hit."""
        tk = lambda t: (t.data_ptr(), t._version, tuple(t.shape), t.dtype, t.device)
        key = (tk(edge_index), tk(edge_type), int(num_nodes))
        hit = self._plans.get(key)
        if hit is not None:
            return hit[0]
        rel = relation_ids(edge_type, self.num_relations)
        R = self.num_relations
        plans = [RgcnPlan(edge_index, rel, num_nodes, r0, min(2, R - r0)) for r0 in range(0, R, 2)]
        if len(self._plans) >= 4:
            self._plans.pop(next(iter(self._plans)))
        self._plans[key] = (plans, edge_index, edge_type)    # the keyed tensors stay alive, so their addresses are not recycled
        return plans

    def _convs(self):
        return [getattr(self, f"conv_{s}_{g}") for g in "ifco" for s in "xh"]

    def _rows_packed(self):
        """(w [4 Co, nb], b [4 Co]) of stmp_lstm_rows_fwd: per gate, block 0 holds the roots and block 1 + r relation r's weights, each
        transposed to (out, in); b = bias_x + bias_h; no peepholes.  One pack launch per parameter change."""
        def build():
            def blocks(c):
                return torch.cat([c.root.unsqueeze(0), c.relation_weights()]).transpose(1, 2)     # (R + 1, out, in)
            cx = [getattr(self, f"conv_x_{g}") for g in "ifco"]
            ch = [getattr(self, f"conv_h_{g}") for g in "ifco"]
            wx = torch.stack([blocks(c) for c in cx])
            wh = torch.stack([blocks(c) for c in ch])
            bx, bh = torch.stack([c.bias for c in cx]), torch.stack([c.bias for c in ch])
            return ops.lstm_rows_pack_weights(_lib.LSTM_GCONV, self.num_relations, self.in_channels, wx, wh, bx, bh, torch.zeros_like(bx))
        return self._rows_pack.get(list(self.parameters()), build)

    def _rows_spec(self):
        """(spec, params) of ops.lstm_rows_train: the block of the packed weight / bias gradient that each parameter receives.  The
        relation weights are autograd views (weight[r]) or products (comp @ V) of the parameters, so autograd carries their blocks on to
        weight and comp: dV_b = sum_r comp[r, b] dW_r, dcomp[r, b] = <dW_r, V_b>."""
        spec, params = [], []
        Ci, Co, R = self.in_channels, self.out_channels, self.num_relations
        C = Ci + Co
        for gi, g in enumerate("ifco"):
            row = gi * Co
            for s, off, width in (("x", 0, Ci), ("h", Ci, Co)):
                c = getattr(self, f"conv_{s}_{g}")
                spec.append(("wt", row, Co, off, width))
                params.append(c.root)
                for r, W in enumerate(c.relation_weights().unbind(0)):
                    spec.append(("wt", row, Co, (1 + r) * C + off, width))
                    params.append(W)
                spec.append(("b", row, Co))
                params.append(c.bias)
        return spec, params

    def _rows_ok(self, plans, X, H, C, training):
        """The row-split route: 2-D float32 X, in_channels <= 16, 32 channels with one or two relations or 64 with one, H and C None or
        (N, out_channels) float32; training calls also need `fused_training`."""
        Co, R = self.out_channels, self.num_relations
        if X.dim() != 2 or X.dtype != torch.float32 or self.in_channels > 16 or len(plans) != 1:
            return False
        if not ((Co == 32 and R in (1, 2)) or (Co == 64 and R == 1)):
            return False
        if any(S is not None and (S.shape != (X.size(0), Co) or S.dtype != torch.float32) for S in (H, C)):
            return False
        if training and not self.fused_training:
            return False
        return ops.lstm_rows_supported(plans[0], _lib.LSTM_GCONV, R, self.in_channels, Co)

    def _conv(self, c, plans, x):
        """One RGCNConv op for op: x @ root + bias + sum_r mean_r(x) @ W_r."""
        out = torch.matmul(x, c.root) + c.bias
        W = c.relation_weights()
        for r in range(self.num_relations):
            out = out + torch.matmul(ops.spmm(plans[r // 2], r % 2, x), W[r])
        return out

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_type: torch.Tensor,
                H: torch.FloatTensor = None, C: torch.FloatTensor = None):
        _require_cuda(X, "X")
        N, Co = X.size(-2), self.out_channels
        plans = self._relation_plans(edge_index, edge_type, N)
        needs_grad = torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or X.requires_grad
                                                  or (H is not None and H.requires_grad) or (C is not None and C.requires_grad))
        if self._rows_ok(plans, X, H, C, needs_grad):      # the row-split LSTM cell (stmp_lstm_rows_*): one launch per step
            w, b = self._rows_packed()
            if needs_grad:
                spec, params = self._rows_spec()
                return ops.lstm_rows_train(plans[0], _lib.LSTM_GCONV, self.num_relations, X, H, C, w, b, None, spec, params)
            return ops.lstm_rows_fwd(plans[0], _lib.LSTM_GCONV, self.num_relations, X, H, C, w, b, None)
        if H is None:
            H = torch.zeros(*X.shape[:-1], Co, device=X.device, dtype=X.dtype)
        if C is None:
            C = torch.zeros(*X.shape[:-1], Co, device=X.device, dtype=X.dtype)

        def gate(g):
            return self._conv(getattr(self, f"conv_x_{g}"), plans, X) + self._conv(getattr(self, f"conv_h_{g}"), plans, H)
        I, F = torch.sigmoid(gate("i")), torch.sigmoid(gate("f"))
        Cn = F * C + I * torch.tanh(gate("c"))
        O = torch.sigmoid(gate("o"))                        # no peephole: O does not read the new cell state
        return O * torch.tanh(Cn), Cn
