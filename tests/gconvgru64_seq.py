"""The reference's tutorial model at 64 hidden channels -- GConvGRU(F, 64, K), ReLU, Linear(64, 1) -- on the WikiMaths fixture of
tests/wikimaths_seq.py and on the in-tree chickenpox split, shared by tests/golden/make_goldens_gconvgru64.py, the CPU and GPU tests of the
64-wide row-split cell and tests/perf/bench_gconvgru_wikimaths.py."""
import gzip
import io
import os

import torch

from pytorch_geometric_temporal_b200.nn.recurrent import GConvGRU

WIDTH = 64


class RecurrentGCN64(torch.nn.Module):
    """The tutorial's model at 64 channels (state_dict keys recurrent.*, linear.*); `gru` is the GConvGRU class (this package's or the
    reference's)."""

    def __init__(self, node_features, K, normalization="sym", gru=GConvGRU):
        super().__init__()
        self.recurrent = gru(node_features, WIDTH, K, normalization=normalization)
        self.linear = torch.nn.Linear(WIDTH, 1)


def carried_h0(n):
    """H0 of the carried case: exact multiples of 1/16 in [-0.5, 0.5], computed rather than stored."""
    i = torch.arange(n).unsqueeze(1) * 7 + torch.arange(WIDTH).unsqueeze(0) * 13
    return ((i % 17) - 8).float() / 16


def load(golden_dir):
    """The 64-wide cases (tests/golden/gconvgru64.pt.gz), each with its model state, predictions, costs and gradients."""
    with gzip.open(os.path.join(golden_dir, "gconvgru64.pt.gz"), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def model_for(c, device="cpu", fused=True, node_features=14):
    m = RecurrentGCN64(node_features, c["K"], c["normalization"])
    m.load_state_dict(c["state"])
    m.recurrent.fused_training = fused
    return m.to(device)


def run_wikimaths(m, X, Y, ei, ew, lam=None, H0=None, backward=True):
    """(predictions (S, N, 1), per-snapshot costs (S,)): H0 None -- the tutorial, one backward per snapshot; else the state carried from H0
    and the mean cost backpropagated once."""
    h, total, outs, losses = H0, 0, [], []
    for t in range(X.shape[0]):
        if H0 is None:
            hh = m.recurrent(X[t], ei, ew, lambda_max=lam)
        else:
            h = hh = m.recurrent(X[t], ei, ew, h, lambda_max=lam)
        y = m.linear(torch.relu(hh))
        cost = torch.mean((y.squeeze() - Y[t]) ** 2)
        outs.append(y.detach())
        losses.append(cost.detach())
        if H0 is None and backward:
            cost.backward()
        total = total + cost
    if H0 is not None and backward:
        (total / X.shape[0]).backward()
    return torch.stack(outs), torch.stack(losses)


def run_chickenpox(m, X, Y, ei, ew):
    """The chickenpox example's epoch: H = None at every snapshot, the cumulative MSE averaged over the snapshots -> (predictions, cost)."""
    cost, outs = 0, []
    for t in range(X.shape[0]):
        y = m.linear(torch.relu(m.recurrent(X[t], ei, ew)))
        outs.append(y.detach())
        cost = cost + torch.mean((y - Y[t]) ** 2)
    return torch.stack(outs), cost / X.shape[0]
