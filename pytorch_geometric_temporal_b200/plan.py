"""GraphPlan: Python owner of an `stmp_plan` (cached, normalised graph operators on the device).

Replaces the per-call renormalisation in the reference (dcrnn.py:59-77 dense adjacency + nonzero,
PyG get_laplacian/gcn_norm on every ChebConv/GCNConv call) and BatchedDCRNN's `torch.equal`
freshness test (dcrnn.py:446-447, a device sync per forward): freshness is decided on the host from
(data_ptr, _version, shape) of edge_index / edge_weight.
"""
import ctypes
from typing import Optional

import torch

from . import _lib


def _require_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(
            f"{name} is on {t.device}: pytorch_geometric_temporal_b200 runs the hot path on CUDA only "
            "(hand-written sm_90a kernels, no CPU fallback).")


class GraphPlan:
    def __init__(self, flavor: int, edge_index: torch.Tensor, edge_weight: Optional[torch.Tensor], num_nodes: int,
                 normalization=None, lambda_max: Optional[float] = None, flags: int = 0,
                 lambda_node: Optional[torch.Tensor] = None):
        _require_cuda(edge_index, "edge_index")
        if edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError(f"edge_index must have shape [2, E], got {tuple(edge_index.shape)}")
        if normalization not in _lib.NORM_CODE:
            raise AssertionError("Invalid normalization")  # astgcn.py:62
        ei = edge_index.to(torch.int64).contiguous()
        ew = None
        if edge_weight is not None:
            _require_cuda(edge_weight, "edge_weight")
            ew = edge_weight.detach().to(torch.float32).contiguous()
            if ew.numel() != ei.size(1):
                raise RuntimeError(f"edge_weight has {ew.numel()} entries for {ei.size(1)} edges")
        self.flavor, self.num_nodes, self.num_edges = flavor, int(num_nodes), int(ei.size(1))
        self.device = ei.device
        self._h = ctypes.c_void_p()
        lam = -1.0 if lambda_max is None else float(lambda_max)
        with torch.cuda.device(ei.device):
            if lambda_node is not None:      # per-graph lambda_max of a multi-graph mini-batch, already expanded to nodes
                ln = lambda_node.detach().to(device=ei.device, dtype=torch.float32).contiguous()
                if ln.numel() != self.num_nodes:
                    raise RuntimeError(f"lambda_max[batch] has {ln.numel()} entries for {self.num_nodes} nodes")
                rc = _lib.lib().stmp_plan_create_pergraph(flavor, self.num_nodes, self.num_edges, _lib.ptr(ei), _lib.ptr(ew),
                                                          _lib.NORM_CODE[normalization], _lib.ptr(ln), flags, _lib.stream_ptr(),
                                                          ctypes.byref(self._h))
            else:
                rc = _lib.lib().stmp_plan_create(flavor, self.num_nodes, self.num_edges, _lib.ptr(ei), _lib.ptr(ew),
                                                 _lib.NORM_CODE[normalization], lam, flags, _lib.stream_ptr(),
                                                 ctypes.byref(self._h))
        _lib.check(rc)
        self.n_ops = _lib.lib().stmp_plan_num_ops(self._h)

    @property
    def handle(self):
        return self._h

    def nnz(self, op: int = 0) -> int:
        return int(_lib.lib().stmp_plan_nnz(self._h, op))

    def export(self, op: int = 0, transposed: bool = False):
        """(rowptr, col, val, eid) as torch tensors -- test/introspection helper."""
        n, nnz = self.num_nodes, self.nnz(op)
        rowptr = torch.empty(n + 1, dtype=torch.int32, device=self.device)
        col = torch.empty(nnz, dtype=torch.int32, device=self.device)
        val = torch.empty(nnz, dtype=torch.float32, device=self.device)
        eid = torch.empty(nnz, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().stmp_plan_export(self._h, op, int(transposed), _lib.ptr(rowptr), _lib.ptr(col),
                                                   _lib.ptr(val), _lib.ptr(eid), _lib.stream_ptr()))
        return rowptr, col, val, eid

    def graph_image(self, n_ops: int):
        """The wgmma kernel's shared-memory image of the first `n_ops` operators as a CPU uint8 tensor, or None when the
        plan has none -- test/introspection helper."""
        size = int(_lib.lib().stmp_plan_graph_image(self._h, n_ops, None, 0))
        if size <= 0:
            return None
        buf = torch.empty(size, dtype=torch.uint8)
        with torch.cuda.device(self.device):
            rc = int(_lib.lib().stmp_plan_graph_image(self._h, n_ops, ctypes.c_void_p(buf.data_ptr()), size))
        if rc < 0:
            _lib.check(-rc)
        return buf

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().stmp_plan_destroy(h)
            except Exception:
                pass
            self._h = None


class RgcnPlan(GraphPlan):
    """The relation-masked mean operators of PyG RGCNConv (STMP_FLAVOR_RGCN) for relations rel0 .. rel0 + n_rel - 1 (n_rel 1 or 2):
    operator k aggregates the edges whose `rel` (int64, one relation id per edge; anything else matches no operator) is rel0 + k."""

    def __init__(self, edge_index: torch.Tensor, rel: torch.Tensor, num_nodes: int, rel0: int, n_rel: int):
        _require_cuda(edge_index, "edge_index")
        if edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError(f"edge_index must have shape [2, E], got {tuple(edge_index.shape)}")
        ei = edge_index.to(torch.int64).contiguous()
        rel = rel.to(device=ei.device, dtype=torch.int64).contiguous()
        if rel.numel() != ei.size(1):
            raise RuntimeError(f"edge_type has {rel.numel()} entries for {ei.size(1)} edges")
        self.flavor, self.num_nodes, self.num_edges = _lib.FLAVOR_RGCN, int(num_nodes), int(ei.size(1))
        self.device = ei.device
        self._h = ctypes.c_void_p()
        with torch.cuda.device(ei.device):
            rc = _lib.lib().stmp_plan_create_rgcn(self.num_nodes, self.num_edges, _lib.ptr(ei), _lib.ptr(rel), int(rel0), int(n_rel),
                                                  _lib.stream_ptr(), ctypes.byref(self._h))
        _lib.check(rc)
        self.n_ops = _lib.lib().stmp_plan_num_ops(self._h)


class BipartitePlan(RgcnPlan):
    """PyG SAGEConv's mean aggregation from `num_src` source rows onto `num_dst` destination rows (one edge type of a heterogeneous
    graph): an STMP_FLAVOR_RGCN plan of one relation holding every edge, built on max(num_src, num_dst) nodes, so its rows < num_dst are
    the destinations and its columns are < num_src.  Sources are checked against num_src and destinations against num_dst here (one host
    sync, a setup path); anything out of range raises RuntimeError."""

    def __init__(self, edge_index: torch.Tensor, num_src: int, num_dst: int):
        _require_cuda(edge_index, "edge_index")
        if edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError(f"edge_index must have shape [2, E], got {tuple(edge_index.shape)}")
        ei = edge_index.to(torch.int64)
        if ei.size(1) and bool(((ei < 0).any(1) | (ei.max(1).values >= torch.tensor([num_src, num_dst], device=ei.device))).any()):
            raise RuntimeError(f"edge_index out of range for {num_src} source and {num_dst} destination nodes")
        super().__init__(ei, torch.zeros(ei.size(1), dtype=torch.int64, device=ei.device), max(int(num_src), int(num_dst), 1), 0, 1)
        self.num_src, self.num_dst = int(num_src), int(num_dst)


class GatedPlan(GraphPlan):
    """PyG GatedGraphConv's aggregation operator (STMP_FLAVOR_GATED) for `aggr` ("add", "mean" or "max"): every edge in edge order,
    value w_e (add, max) or w_e / (the destination's count of in-edges) (mean); edge_weight None means ones."""

    def __init__(self, edge_index: torch.Tensor, edge_weight: Optional[torch.Tensor], num_nodes: int, aggr: str):
        _require_cuda(edge_index, "edge_index")
        if edge_index.dim() != 2 or edge_index.size(0) != 2:
            raise ValueError(f"edge_index must have shape [2, E], got {tuple(edge_index.shape)}")
        ei = edge_index.to(torch.int64).contiguous()
        ew = None
        if edge_weight is not None:
            _require_cuda(edge_weight, "edge_weight")
            ew = edge_weight.detach().to(torch.float32).reshape(-1).contiguous()
            if ew.numel() != ei.size(1):
                raise RuntimeError(f"edge_weight has {ew.numel()} entries for {ei.size(1)} edges")
        self.flavor, self.num_nodes, self.num_edges, self.aggr = _lib.FLAVOR_GATED, int(num_nodes), int(ei.size(1)), aggr
        self.device = ei.device
        self._h = ctypes.c_void_p()
        with torch.cuda.device(ei.device):
            rc = _lib.lib().stmp_plan_create_gated(self.num_nodes, self.num_edges, _lib.ptr(ei), _lib.ptr(ew), _lib.AGGR_CODE[aggr],
                                                   _lib.stream_ptr(), ctypes.byref(self._h))
        _lib.check(rc)
        self.n_ops = _lib.lib().stmp_plan_num_ops(self._h)


class PlanCache:
    """Per-module cache keyed on the identity/version of the graph tensors (no device sync)."""

    def __init__(self, max_entries: int = 4):
        self._entries = {}
        self._max = max_entries

    @staticmethod
    def _tkey(t):
        return None if t is None else (t.data_ptr(), t._version, tuple(t.shape), t.dtype, t.device)

    def get(self, flavor, edge_index, edge_weight, num_nodes, normalization=None, lambda_max=None, flags=0, batch=None) -> GraphPlan:
        """`lambda_max`: None, a host scalar / 0-d tensor, or -- with the node->graph vector `batch` -- one value per graph
        (PyG: `lambda_max[batch[edge_index[0]]]`)."""
        lam, lam_node, extra = None, None, ()
        if lambda_max is not None:
            if torch.is_tensor(lambda_max) and lambda_max.numel() > 1:
                if batch is None:
                    raise ValueError("a lambda_max vector needs the `batch` vector of the mini-batch (one graph id per node)")
                lam_node = lambda_max.to(torch.float32)[batch]
                extra = (self._tkey(lambda_max), self._tkey(batch))
            else:
                lam = float(lambda_max)  # scalar lambda_max (host value or 0-d tensor; a sync only if it is a tensor)
        key = (flavor, self._tkey(edge_index), self._tkey(edge_weight), int(num_nodes), normalization, lam, flags) + extra
        return self._lookup(key, lambda: GraphPlan(flavor, edge_index, edge_weight, num_nodes, normalization, lam, flags,
                                                   lambda_node=lam_node),
                            (edge_index, edge_weight, lambda_max if extra else None, batch if extra else None))

    def get_gated(self, edge_index, edge_weight, num_nodes, aggr) -> GatedPlan:
        """The GatedPlan of `aggr` ("add", "mean" or "max") for this graph."""
        key = (_lib.FLAVOR_GATED, self._tkey(edge_index), self._tkey(edge_weight), int(num_nodes), aggr)
        return self._lookup(key, lambda: GatedPlan(edge_index, edge_weight, num_nodes, aggr), (edge_index, edge_weight))

    def get_bipartite(self, edge_index, num_src, num_dst) -> BipartitePlan:
        """The BipartitePlan of one edge type of a heterogeneous graph."""
        key = ("bipartite", self._tkey(edge_index), int(num_src), int(num_dst))
        return self._lookup(key, lambda: BipartitePlan(edge_index, num_src, num_dst), (edge_index,))

    def _lookup(self, key, make, keep):
        hit = self._entries.get(key)
        if hit is not None:
            return hit[0]
        plan = make()
        if len(self._entries) >= self._max:
            self._entries.pop(next(iter(self._entries)))
        # keep the keyed tensors alive so their addresses cannot be recycled while the entry exists
        self._entries[key] = (plan, *keep)
        return plan
