"""StaticHeteroGraphTemporalSignal -- drop-in for the reference's signal/static_hetero_graph_temporal_signal.py, and HeteroData, the part of
PyG's heterogeneous snapshot its users read: `data[node_type]` / `data[edge_type]` stores, `node_types`, `edge_types`, `node_stores`,
`edge_stores`, `x_dict`, `edge_index_dict`, `metadata()` and `.to(device)`.

As StaticGraphTemporalSignal does for one graph, the static edge tensors are converted once and every snapshot hands out the same
tensor objects, and a snapshot's `.to(device)` reuses one device copy of each, memoised on its signal for every edge tensor it has: the reference mints new edge tensors on every
snapshot, which would make HeteroGCLSTM rebuild its plans, with a host sync, on every step of a loop."""
from typing import Dict, Sequence, Tuple, Union

import numpy as np
import torch

from .data import _memo_to

_GRAPH_KEYS = ("edge_index", "edge_attr")


class _Store(dict):
    """Attribute view of one node or edge type's tensors."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k) from None

    def __setattr__(self, k, v):
        self[k] = v


class HeteroData(object):
    def __init__(self):
        self._nodes, self._edges = {}, {}
        self._device_copies = None       # a signal's snapshots share its memo of static edge tensors' device copies

    def _graph_to(self, v, device, non_blocking):
        if self._device_copies is None:
            return _memo_to(v, device, non_blocking)
        key = (id(v), v._version, str(device))
        hit = self._device_copies.get(key)
        if hit is None or hit[0] is not v:
            hit = self._device_copies[key] = (v, v.to(device, non_blocking=non_blocking))
        return hit[1]

    def __getitem__(self, key):
        if isinstance(key, tuple):
            return self._edges.setdefault(key, _Store())
        return self._nodes.setdefault(key, _Store())

    @property
    def node_types(self):
        return list(self._nodes)

    @property
    def edge_types(self):
        return list(self._edges)

    @property
    def node_stores(self):
        return list(self._nodes.values())

    @property
    def edge_stores(self):
        return list(self._edges.values())

    def _collect(self, stores, name):
        return {k: s[name] for k, s in stores.items() if name in s}

    @property
    def x_dict(self):
        return self._collect(self._nodes, "x")

    @property
    def y_dict(self):
        return self._collect(self._nodes, "y")

    @property
    def edge_index_dict(self):
        return self._collect(self._edges, "edge_index")

    @property
    def edge_attr_dict(self):
        return self._collect(self._edges, "edge_attr")

    def metadata(self):
        return self.node_types, self.edge_types

    def to(self, device, non_blocking=False):
        out = HeteroData()
        out._device_copies = self._device_copies
        for src, dst, graph in ((self._nodes, out._nodes, False), (self._edges, out._edges, True)):
            for k, s in src.items():
                dst[k] = _Store({n: (self._graph_to(v, device, non_blocking) if graph and n in _GRAPH_KEYS
                                     else v.to(device, non_blocking=non_blocking)) if torch.is_tensor(v) else v for n, v in s.items()})
        return out

    def cuda(self, device=None, non_blocking=False):
        return self.to(torch.device("cuda" if device is None else device), non_blocking)

    def __repr__(self):
        return f"HeteroData(node_types={self.node_types}, edge_types={self.edge_types})"


Edge_Index = Union[Dict[Tuple[str, str, str], np.ndarray], None]
Edge_Weight = Union[Dict[Tuple[str, str, str], np.ndarray], None]
Node_Features = Sequence[Union[Dict[str, np.ndarray], None]]
Targets = Sequence[Union[Dict[str, np.ndarray], None]]


def _typed(d):
    """The reference's per-type conversion: float arrays to FloatTensor, integer arrays to LongTensor, others as they are; None dropped."""
    if d is None:
        return None
    return {k: torch.FloatTensor(v) if v.dtype.kind == "f" else torch.LongTensor(v) if v.dtype.kind == "i" else v
            for k, v in d.items() if v is not None}


class StaticHeteroGraphTemporalSignal(object):
    def __init__(self, edge_index_dict: Edge_Index, edge_weight_dict: Edge_Weight, feature_dicts: Node_Features, target_dicts: Targets,
                 **kwargs):
        self.edge_index_dict, self.edge_weight_dict = edge_index_dict, edge_weight_dict
        self.feature_dicts, self.target_dicts = feature_dicts, target_dicts
        self.additional_feature_keys = []
        for key, value in kwargs.items():
            setattr(self, key, value)
            self.additional_feature_keys.append(key)
        assert len(self.feature_dicts) == len(self.target_dicts), "Temporal dimension inconsistency."
        for key in self.additional_feature_keys:
            assert len(self.target_dicts) == len(getattr(self, key)), "Temporal dimension inconsistency."
        self.snapshot_count = len(self.feature_dicts)
        self._graph = None
        self._device_copies = {}         # (id, _version, device) of a static edge tensor -> (tensor, its device copy), one per tensor
        self.t = 0

    def _static_graph(self):
        """(edge_index tensors, edge_weight tensors), converted once and shared by every snapshot."""
        if self._graph is None:
            ei = None if self.edge_index_dict is None else {k: torch.LongTensor(v) for k, v in self.edge_index_dict.items()}
            ew = None if self.edge_weight_dict is None else {k: torch.FloatTensor(v) for k, v in self.edge_weight_dict.items()}
            self._graph = (ei, ew)
        return self._graph

    def _get_features(self, time_index: int):
        d = self.feature_dicts[time_index]
        return None if d is None else {k: torch.FloatTensor(v) for k, v in d.items() if v is not None}

    def __getitem__(self, time_index: Union[int, slice]):
        if isinstance(time_index, slice):
            return StaticHeteroGraphTemporalSignal(self.edge_index_dict, self.edge_weight_dict, self.feature_dicts[time_index],
                                                   self.target_dicts[time_index],
                                                   **{key: getattr(self, key)[time_index] for key in self.additional_feature_keys})
        x_dict = self._get_features(time_index)
        edge_index_dict, edge_weight_dict = self._static_graph()
        y_dict = _typed(self.target_dicts[time_index])
        snapshot = HeteroData()
        snapshot._device_copies = self._device_copies
        for name, d in (("x", x_dict), ("edge_index", edge_index_dict), ("edge_attr", edge_weight_dict), ("y", y_dict)):
            for key, value in (d or {}).items():
                snapshot[key][name] = value
        for feature_name in self.additional_feature_keys:
            for key, value in (_typed(getattr(self, feature_name)[time_index]) or {}).items():
                snapshot[key][feature_name] = value
        return snapshot

    def __next__(self):
        if self.t < len(self.feature_dicts):
            snapshot = self[self.t]
            self.t = self.t + 1
            return snapshot
        self.t = 0
        raise StopIteration

    def __iter__(self):
        self.t = 0
        return self
