"""The LSTM tutorial loop of tests/golden/make_goldens_lstm.py on any module pair, shared by the golden generator, the CPU and GPU tests and
tests/perf/bench_lstm_train.py: examples/recurrent/gconvlstm_example.py's and gclstm_example.py's model (GConvLSTM or GCLSTM(F, 32, K),
ReLU, Linear(32, 1)) over a sequence of snapshots with H and C carried from None (or from leaf H0 / C0), a cumulative MSE divided by the
number of snapshots and one backward at the end."""
import gzip
import io
import os

import torch

from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvLSTM
from gconvgru_seq import chickenpox_train_split
import wikimaths_seq

MODULES = {"gconvlstm": GConvLSTM, "gclstm": GCLSTM}
FIXTURE = "lstm_rows.pt.gz"
WIKI_SNAPSHOTS = 3


class RecurrentGCN(torch.nn.Module):
    """The examples' model (state_dict keys recurrent.*, linear.*)."""

    def __init__(self, cls, node_features, K, normalization="sym"):
        super().__init__()
        self.recurrent = cls(node_features, 32, K, normalization=normalization)
        self.linear = torch.nn.Linear(32, 1)


def carried_state(n, a, b, m):
    """A leaf state of exact multiples of 1/16 in [-0.5, 0.5], computed rather than stored."""
    i = torch.arange(n).unsqueeze(1) * a + torch.arange(32).unsqueeze(0) * b
    return ((i % m) - (m // 2)).float() / 16


def data(name, golden_dir):
    """(edge_index, edge_weight, X (S, N, F), Y (S, N), H0, C0) of a data set: the chickenpox tutorial split, the METR-LA-shaped sequence
    (12 steps carried from a computed leaf H0 / C0) or the first snapshots of the WikiMaths tutorial."""
    if name == "chickenpox":
        ei, ew, X, Y = chickenpox_train_split()
        return ei, ew, X, Y, None, None
    if name == "metr_la":
        ei, ew, series = synthetic.metr_la_like(0, 64)
        X = torch.from_numpy(series[3:15].copy())                         # (12, 207, 2)
        Y = torch.from_numpy(series[4:16, :, 0].copy())                   # next step's first feature
        return torch.from_numpy(ei), torch.from_numpy(ew), X, Y, carried_state(207, 7, 13, 17), carried_state(207, 5, 11, 19)
    g = wikimaths_seq.load(golden_dir)
    return g["edge_index"], g["edge_weight"], g["X"][:WIKI_SNAPSHOTS], g["Y"][:WIKI_SNAPSHOTS], None, None


def load(golden_dir):
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def model_for(g, case, device="cpu", fused=True):
    c = g["cases"][case]
    m = RecurrentGCN(MODULES[c["module"]], c["F"], c["K"], c["normalization"])
    m.load_state_dict(g["states"][c["state"]])
    m.recurrent.fused_training = fused
    return m.to(device)


def run(m, ei, ew, X, Y, lambda_max=None, H0=None, C0=None, device="cpu"):
    """(every step's prediction (S, N, 1), cost): H and C carried from H0 / C0 (None: the module's zeros), cumulative MSE / S."""
    ei, ew, X, Y = ei.to(device), ew.to(device), X.to(device), Y.to(device)
    lam = None if lambda_max is None else lambda_max.to(device)
    h, c, cost, outs = H0, C0, 0, []
    for t in range(X.shape[0]):
        h, c = m.recurrent(X[t], ei, ew, h, c, lambda_max=lam)
        y = m.linear(torch.relu(h))
        outs.append(y)
        cost = cost + torch.mean((y - Y[t]) ** 2)      # (N, 1) - (N,) broadcasts, as in the examples' cost
    return torch.stack(outs), cost / X.shape[0]


def run_case_data(m, name, golden_dir, lambda_max=None, device="cpu", state_grad=True):
    """run() on a data set (see data()); H0 / C0, when the data set has them, are leaves that require grad with `state_grad`.
    Returns (outs, cost, H0, C0)."""
    ei, ew, X, Y, H0, C0 = data(name, golden_dir)
    if H0 is not None:
        H0, C0 = H0.to(device).requires_grad_(state_grad), C0.to(device).requires_grad_(state_grad)
    outs, cost = run(m, ei, ew, X, Y, lambda_max, H0, C0, device)
    return outs, cost, H0, C0


def run_case(m, g, case, golden_dir, device="cpu", state_grad=True):
    """run_case_data() on a fixture case's data set and lambda_max."""
    c = g["cases"][case]
    return run_case_data(m, c["data"], golden_dir, c.get("lambda_max"), device, state_grad)
