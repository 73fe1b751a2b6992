"""Shared pieces of the ChebConv cells: parameter holders with PyG's state_dict layout and the shared
Chebyshev basis (one set of SpMMs per step instead of one per gate)."""
import math

import torch

from ... import _lib, ops
from ...plan import PlanCache


def glorot_(t: torch.Tensor):
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)


class _Lin(torch.nn.Module):
    """PyG Linear(in, out, bias=False, weight_initializer='glorot'): key `weight` (out,in)."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.empty(out_channels, in_channels))
        glorot_(self.weight)


class ChebParams(torch.nn.Module):
    """Parameter holder with ChebConv's state_dict keys: `lins.{k}.weight (out,in)`, `bias (out)`."""

    def __init__(self, in_channels, out_channels, K, bias=True):
        super().__init__()
        assert K > 0
        self.in_channels, self.out_channels, self.K = in_channels, out_channels, K
        self.lins = torch.nn.ModuleList([_Lin(in_channels, out_channels) for _ in range(K)])
        if bias:
            self.bias = torch.nn.Parameter(torch.zeros(out_channels))
        else:
            self.register_parameter("bias", None)

    def stacked(self):
        """(K*in, out): rows of block k are lins[k].weight^T."""
        return torch.cat([l.weight.t() for l in self.lins], dim=0)


class ChebPlanMixin:
    """lambda_max semantics of PyG ChebConv (current): None => 2*max(w_hat) (computed on the device
    inside the plan); a scalar/0-d tensor => used as is; a per-graph vector together with the node->graph
    `batch` vector of a multi-graph mini-batch => `lambda_max[batch[edge_index[0]]]` inside the plan."""

    def _init_plans(self):
        self._plans = PlanCache()
        self._lam_cache = {}

    def _lambda_value(self, lambda_max):
        if lambda_max is None:
            return None
        if torch.is_tensor(lambda_max):
            if lambda_max.numel() != 1:
                raise ValueError("per-graph lambda_max needs a `batch` vector; only scalar lambda_max is supported")
            key = (lambda_max.data_ptr(), lambda_max._version, lambda_max.device)
            hit = self._lam_cache.get(key)
            if hit is None:
                if len(self._lam_cache) > 8:
                    self._lam_cache.clear()
                hit = (float(lambda_max), lambda_max)  # one sync per distinct tensor, kept alive with the key
                self._lam_cache[key] = hit
            return hit[0]
        return float(lambda_max)

    def _cheb_plan(self, edge_index, edge_weight, num_nodes, normalization, lambda_max, batch=None):
        if normalization not in (None, "sym", "rw"):
            raise AssertionError("Invalid normalization")
        if batch is not None and torch.is_tensor(lambda_max) and lambda_max.numel() > 1:
            return self._plans.get(_lib.FLAVOR_CHEB, edge_index, edge_weight, num_nodes, normalization, lambda_max, batch=batch)
        return self._plans.get(_lib.FLAVOR_CHEB, edge_index, edge_weight, num_nodes, normalization,
                               self._lambda_value(lambda_max))


def broadcast_states(X: torch.Tensor, states, out_channels: int):
    """(X, [S, ..]) broadcast to one leading shape, a state None becoming zeros of it: the reference sums conv(X), conv(H) and w_c * C
    elementwise, so an (N, out) state is shared by every window of a (B, N, F) batch.  The kernels behind the basis buffer walk the
    rows of X and of every state alike, so each must hold all of them; `broadcast_to` keeps the gradient of a shared state the sum
    over the batch."""
    lead = torch.broadcast_shapes(X.shape[:-1], *(S.shape[:-1] for S in states if S is not None))
    out = [torch.zeros(*lead, out_channels, device=X.device, dtype=X.dtype) if S is None else S.broadcast_to(*lead, out_channels)
           for S in states]
    return X.broadcast_to(*lead, X.size(-1)), out


def cheb_basis(plan, U: torch.Tensor, K: int):
    """[T_0, .., T_{K-1}](U): T_0=U, T_1=L^U, T_k = 2 L^ T_{k-1} - T_{k-2}."""
    T = [U]
    if K > 1:
        T.append(ops.spmm(plan, 0, U))
    for _ in range(2, K):
        T.append(ops.spmm(plan, 0, T[-1], alpha=2.0, z=T[-2], beta=-1.0))
    return T


class ChebConv(ChebParams, ChebPlanMixin):
    """PyG ChebConv as a layer (ctor sites stgcn.py:108-114, mstgcn.py:33): `forward(x, edge_index, edge_weight=None,
    batch=None, lambda_max=None)`, x (N,F) or (B,N,F) -- every leading batch row shares the cached operator, so the
    reference's Python loops over (b, t) slices (stgcn.py:151-153) become the batch axis of one SpMM launch per hop,
    followed by one GEMM over the stacked basis."""

    def __init__(self, in_channels: int, out_channels: int, K: int, normalization="sym", bias: bool = True, **kwargs):
        super().__init__(in_channels, out_channels, K, bias)
        assert normalization in (None, "sym", "rw"), "Invalid normalization"
        self.normalization = normalization
        self._init_plans()

    def forward(self, x, edge_index, edge_weight=None, batch=None, lambda_max=None):
        if self.K > 1:
            plan = self._cheb_plan(edge_index, edge_weight, x.size(-2), self.normalization, lambda_max, batch)
            S = torch.cat(cheb_basis(plan, x, self.K), dim=-1)
        else:
            S = x                                                        # K=1: no propagation at all
        out = torch.matmul(S, self.stacked())
        return out if self.bias is None else out + self.bias

    def __repr__(self):
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, K={self.K}, normalization={self.normalization})"
