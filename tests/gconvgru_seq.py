"""The GConvGRU training loops of tests/golden/make_goldens_gconvgru.py on this package's modules, shared by the CPU and GPU tests and by
tests/perf/bench_gconvgru_train.py: the reference's tutorial model (GConvGRU(F, 32, K), ReLU, Linear(32, 1)) over a sequence of snapshots
with a cumulative-MSE cost, either from H = None at every snapshot (examples/recurrent/gconvgru_example.py) or with the state carried."""
import os

import numpy as np
import torch

from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


class RecurrentGCN(torch.nn.Module):
    """The example's model (state_dict keys recurrent.*, linear.*)."""

    def __init__(self, node_features, K, normalization="sym", bias=True):
        super().__init__()
        self.recurrent = GConvGRU(node_features, 32, K, normalization=normalization, bias=bias)
        self.linear = torch.nn.Linear(32, 1)


def chickenpox_train_split(lags=4, train_ratio=0.2):
    """(edge_index, edge_weight, X (S, 20, lags), Y (S, 20)): the snapshots of temporal_signal_split(dataset, train_ratio=0.2) of the
    in-tree chickenpox data (ChickenpoxDatasetLoader().get_dataset(lags))."""
    z = np.load(os.path.join(ROOT, "pytorch_geometric_temporal_b200", "dataset", "data", "chickenpox.npz"))
    ei = torch.tensor(z["edges"], dtype=torch.int64).T.contiguous()
    ew = torch.ones(ei.shape[1], dtype=torch.float32)
    FX = np.asarray(z["FX"], dtype=np.float32)
    n = FX.shape[0] - lags
    S = int(train_ratio * n)
    X = torch.from_numpy(np.stack([FX[i:i + lags].T for i in range(S)]).copy())
    Y = torch.from_numpy(np.stack([FX[i + lags] for i in range(S)]).copy())
    return ei, ew, X, Y


def model_for(g, device="cpu", fused=True):
    m = RecurrentGCN(g["X"].shape[-1], g["K"], g["normalization"], bias=g.get("bias", True))
    m.load_state_dict(g["state"])
    m.recurrent.fused_training = fused
    return m.to(device)


def run(m, g, device="cpu", H0=None):
    """(every step's prediction (S, N, 1), cost): H = None per snapshot, or the state carried from H0."""
    ei, ew = g["edge_index"].to(device), g["edge_weight"].to(device)
    X, Y = g["X"].to(device), g["Y"].to(device)
    lam = g.get("lambda_max")
    lam = None if lam is None else lam.to(device)
    h, cost, outs = H0, 0, []
    for t in range(X.shape[0]):
        if H0 is None:
            hh = m.recurrent(X[t], ei, ew, lambda_max=lam)
        else:
            h = hh = m.recurrent(X[t], ei, ew, h, lambda_max=lam)
        y = m.linear(torch.relu(hh))
        outs.append(y)
        cost = cost + torch.mean((y - Y[t]) ** 2)      # (N, 1) - (N,) broadcasts, as in the example's cost
    return torch.stack(outs), cost / X.shape[0]
