"""The TGCN training loops of tests/golden/make_goldens_tgcn.py on this package's modules, shared by the CPU and GPU tests: a TGCN2 (or
TGCN) cell called once per step with the hidden state carried, ReLU, then a Linear head."""
import os

import torch

from pytorch_geometric_temporal_b200.nn.recurrent import TGCN, TGCN2


def load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


class SeqModel(torch.nn.Module):
    """BatchedTGCN of the reference's index-batching scripts (state_dict keys tgnn.*, linear.*)."""

    def __init__(self, cell, hidden, out):
        super().__init__()
        self.tgnn = cell
        self.linear = torch.nn.Linear(hidden, out)


def masked_mae(pred, true):
    """The scripts' masked MAE; NaNs are zeroed with torch.where instead of a masked assignment, so that a CUDA graph can capture it."""
    mask = (true != 0).float()
    mask /= mask.mean()
    loss = torch.abs(pred - true) * mask
    return torch.where(loss != loss, torch.zeros_like(loss), loss).mean()


def model_for(g, device="cpu", fused=True):
    """The golden's model, TGCN2(2, 32, 1) + Linear(32, 2) or TGCN(4, 32) + Linear(32, 1), with its weights."""
    chickenpox = "H0" in g
    m = SeqModel(TGCN(4, 32) if chickenpox else TGCN2(2, 32, 1), 32, 1 if chickenpox else 2)
    m.load_state_dict(g["state"])
    m.tgnn.fused_training = fused
    return m.to(device)


def run(m, g, device="cpu", H0=None):
    """One forward over the golden's window: (every step's output, loss).  X (B, N, F, T) with H = None at t = 0 for the METR-LA /
    PEMS-BAY goldens; 24 chickenpox snapshots from the state H0 with the cumulative-MSE cost for the chickenpox golden."""
    ei, ew = g["edge_index"].to(device), g["edge_weight"].to(device)
    X, Y = g["X"].to(device), g["Y"].to(device)
    if "H0" in g:
        h, cost, outs = H0, 0, []
        for t in range(X.shape[0]):
            h = m.tgnn(X[t], ei, ew, h)
            y = m.linear(torch.relu(h))
            outs.append(y)
            cost = cost + torch.mean((y - Y[t]) ** 2)
        return torch.stack(outs), cost / X.shape[0]
    h, outs = None, []
    for t in range(X.shape[-1]):
        h = m.tgnn(X[..., t], ei, ew, h)
        outs.append(m.linear(torch.relu(h)).unsqueeze(1))
    out = torch.cat(outs, dim=1)
    return out, masked_mae(out, Y)
