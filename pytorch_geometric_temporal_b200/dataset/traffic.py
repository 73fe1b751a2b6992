"""Offline METR-LA / PEMS-BAY loaders -- drop-ins for dataset/metr_la.py (:16-237) and dataset/pems_bay.py (:17-246)
(SURVEY 8f rank 3).  Same class names, constructor `(raw_data_dir, index=False)`, `get_dataset(num_timesteps_in,
num_timesteps_out)` and the 7-tuple of `get_index_dataset(...)`.

There is no network here, so nothing is downloaded: `raw_data_dir` must already hold the two arrays of the public
archives -- `adj_mat.npy (N,N)` + `node_values.npy (T,N,F)` for METR-LA, `pems_adj_mat.npy` + `pems_node_values.npy`
for PEMS-BAY (metr_la.py:66-77, pems_bay.py:72-84); a missing file raises FileNotFoundError naming it.

Addition of this package: `get_index_loaders(...)` returns `signal.IndexBatchLoader`s over a series that lives in HBM
(z-scored on the device, metr_la.py:180-190), sharded per rank with DistributedSampler semantics -- the feed the
fused DCRNN sequence kernel consumes without materialising windows."""
import os
from typing import Tuple

import numpy as np
import torch
from torch.utils.data import DataLoader
from torch.utils.data.distributed import DistributedSampler

from ..signal import IndexBatchLoader, IndexDataset, StaticGraphTemporalSignal, index_splits


def dense_to_sparse(adj: torch.Tensor):
    """torch_geometric.utils.dense_to_sparse for one 2-D matrix: row-major order of the non-zeros (metr_la.py:92)."""
    idx = adj.nonzero().t().contiguous()
    return idx, adj[idx[0], idx[1]]


class _TrafficLoader(object):
    _ADJ, _VALUES, _NAME = "", "", ""
    _SPEED_ONLY_TARGET = True         # METR-LA predicts feature 0 (:118); PEMS-BAY keeps every feature (pems_bay.py:125)

    def __init__(self, raw_data_dir=os.path.join(os.getcwd(), "data"), index: bool = False):
        self.index, self.raw_data_dir = index, raw_data_dir
        for f in (self._ADJ, self._VALUES):
            if not os.path.isfile(os.path.join(raw_data_dir, f)):
                raise FileNotFoundError(f"{self._NAME}: {os.path.join(raw_data_dir, f)} not found (offline loader: place the "
                                        f"extracted archive's {self._ADJ} / {self._VALUES} there)")
        if index:
            self.IndexDataset = IndexDataset
        else:
            A, X = self._load_raw()
            means = np.mean(X, axis=(0, 2))
            X = X - means.reshape(1, -1, 1)
            stds = np.std(X, axis=(0, 2))
            X = X / stds.reshape(1, -1, 1)
            self.A, self.X = torch.from_numpy(A), torch.from_numpy(X)

    def _load_raw(self):
        A = np.load(os.path.join(self.raw_data_dir, self._ADJ))
        X = np.load(os.path.join(self.raw_data_dir, self._VALUES)).transpose((1, 2, 0)).astype(np.float32)   # (N,F,T)
        return A, X

    def _get_edges_and_weights(self):
        ei, w = dense_to_sparse(self.A)
        self.edges, self.edge_weights = ei.numpy(), w.numpy()

    def _generate_task(self, num_timesteps_in: int = 12, num_timesteps_out: int = 12):
        span = num_timesteps_in + num_timesteps_out
        feats, targs = [], []
        for i in range(self.X.shape[2] - span + 1):
            feats.append(self.X[:, :, i:i + num_timesteps_in].numpy())
            tgt = self.X[:, 0, i + num_timesteps_in:i + span] if self._SPEED_ONLY_TARGET else self.X[:, :, i + num_timesteps_in:i + span]
            targs.append(tgt.numpy())
        self.features, self.targets = feats, targs

    def get_dataset(self, num_timesteps_in: int = 12, num_timesteps_out: int = 12, device=None) -> StaticGraphTemporalSignal:
        self._get_edges_and_weights()
        self._generate_task(num_timesteps_in, num_timesteps_out)
        return StaticGraphTemporalSignal(self.edges, self.edge_weights, self.features, self.targets, device=device)

    # ---- index batching -------------------------------------------------------------------------------------------
    def _normalised_series(self, allGPU: int):
        """(T,N,F) z-scored series + means/stds (F,), on cuda:allGPU or as numpy (metr_la.py:176-198)."""
        A, data = self._load_raw()
        edges, edge_weights = dense_to_sparse(torch.from_numpy(A))
        if allGPU != -1:
            data = torch.tensor(data, dtype=torch.float).to(f"cuda:{allGPU}")
            means = torch.mean(data, dim=(0, 2), keepdim=True)
            data = data - means
            stds = torch.std(data, dim=(0, 2), keepdim=True)
            data = (data / stds).permute(2, 0, 1)
            means, stds = means.squeeze(), stds.squeeze()
        else:
            means = np.mean(data, axis=(0, 2))
            data = data - means.reshape(1, -1, 1)
            stds = np.std(data, axis=(0, 2))
            data = (data / stds.reshape(1, -1, 1)).transpose((2, 0, 1))
            means, stds = torch.tensor(means, dtype=torch.float), torch.tensor(stds, dtype=torch.float)
        return data, edges, edge_weights, means, stds

    def get_index_dataset(self, lags: int = 12, batch_size: int = 64, shuffle: bool = False, allGPU: int = -1,
                          ratio: Tuple[float, float, float] = (0.7, 0.1, 0.2), world_size: int = -1, ddp_rank: int = -1,
                          dask_batching: bool = False):
        """(train, val, test DataLoaders, edges, edge_weights, means, stds) -- metr_la.py:143-234."""
        if not self.index:
            raise ValueError("get_index_dataset requires 'index=True' in the constructor.")
        data, edges, edge_weights, means, stds = self._normalised_series(allGPU)
        x_train, x_val, x_test = index_splits(data.shape[0], lags, ratio)
        loaders = []
        for idx in (x_train, x_val, x_test):
            ds = self.IndexDataset(idx, data, lags, gpu=not (allGPU == -1), lazy=dask_batching)
            if ddp_rank != -1:
                sampler = DistributedSampler(ds, num_replicas=world_size, rank=ddp_rank, shuffle=shuffle)
                loaders.append(DataLoader(ds, batch_size=batch_size, sampler=sampler))
            else:
                loaders.append(DataLoader(ds, batch_size=batch_size, shuffle=shuffle))
        return loaders[0], loaders[1], loaders[2], edges, edge_weights, means, stds

    def get_index_loaders(self, device, lags: int = 12, batch_size: int = 64, shuffle: bool = False,
                          ratio: Tuple[float, float, float] = (0.7, 0.1, 0.2), world_size: int = 1, rank: int = 0, seed: int = 0):
        """HBM-resident variant: the same splits/normalisation, windows gathered on the device by `stmp_window_gather`
        (or consumed in place by the fused sequence kernel); returns the same 7-tuple shape with IndexBatchLoaders."""
        dev = torch.device(device)
        data, edges, edge_weights, means, stds = self._normalised_series(dev.index if dev.index is not None else 0)
        data = data.contiguous()
        x_train, x_val, x_test = index_splits(data.shape[0], lags, ratio)
        mk = lambda idx, sh: IndexBatchLoader(data, idx, lags, batch_size, shuffle=sh, world_size=world_size, rank=rank, seed=seed)
        return mk(x_train, shuffle), mk(x_val, False), mk(x_test, False), edges.to(dev), edge_weights.to(dev), means, stds


class METRLADatasetLoader(_TrafficLoader):
    """207 loop detectors, Los Angeles, 5-minute readings (dataset/metr_la.py:16-26)."""
    _ADJ, _VALUES, _NAME = "adj_mat.npy", "node_values.npy", "METR-LA"
    _SPEED_ONLY_TARGET = True


class PemsBayDatasetLoader(_TrafficLoader):
    """325 CalTrans PeMS sensors, Bay Area (dataset/pems_bay.py:17-31)."""
    _ADJ, _VALUES, _NAME = "pems_adj_mat.npy", "pems_node_values.npy", "PEMS-BAY"
    _SPEED_ONLY_TARGET = False
