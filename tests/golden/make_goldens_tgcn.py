"""Golden vectors for TGCN training with the hidden state carried from step to step (the loop of the reference's BatchedTGCN index-batching
scripts and of examples/recurrent/tgcn_example.py) from the UNMODIFIED reference modules (same mechanism as make_goldens_r2.py: the
reference imported through oracle/refload.py on top of oracle/stubs).  Run in the build container only:
python tests/golden/make_goldens_tgcn.py [name ...]

The training loops are written here, not copied from the example scripts:
* tgcn2_seq_metr_la_grads  -- TGCN2(2, 32, 1) + Linear(32, 2) over 12 steps (H = None at t = 0, then carried; ReLU before the Linear),
                              8 windows of the METR-LA-shaped series laid out (B, N, F, T), masked-MAE loss with some zero targets:
                              every step's output, the loss and the gradient of every parameter (tgnn.*, linear.*)
* tgcn2_seq_pems_bay_grads -- the same on the PEMS-BAY-shaped graph (325 nodes), 4 windows
* tgcn_chickenpox_seq_grads -- TGCN(4, 32) + Linear(32, 1) over the first 24 chickenpox snapshots (lags = 4) from a user-supplied state
                               H0, cumulative-MSE cost divided by the number of snapshots: outputs, cost, parameter gradients and dL/dH0
Biases are set to non-zero values so that their gradients are exercised.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refload  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def save(name, **kw):
    torch.save(kw, os.path.join(OUT, name + ".pt"))
    print(f"{name}.pt  {os.path.getsize(os.path.join(OUT, name + '.pt')) / 1024:.0f} KB")


def sd(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def _nonzero_biases(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)


def masked_mae(pred, true):
    """The masked MAE of the index-batching scripts: zero targets are masked out, the mask renormalised to mean 1."""
    mask = (true != 0).float()
    mask /= mask.mean()
    loss = torch.abs(pred - true) * mask
    loss[loss != loss] = 0
    return loss.mean()


class _Seq(torch.nn.Module):
    def __init__(self, cell, hidden, out):
        super().__init__()
        self.tgnn = cell
        self.linear = torch.nn.Linear(hidden, out)


def _seq(name, ei, ew, series, B, seed):
    tg = refload.load("nn.recurrent.temporalgcn")
    ei_t, ew_t = torch.from_numpy(ei), torch.from_numpy(ew)
    torch.manual_seed(seed)
    m = _Seq(tg.TGCN2(2, 32, 1), 32, 2)
    _nonzero_biases(m, seed)
    starts = [5 + 17 * i for i in range(B)]
    X = torch.from_numpy(np.stack([series[s:s + 12] for s in starts])).permute(0, 2, 3, 1).contiguous()     # (B, N, F, T)
    Y = torch.from_numpy(np.stack([series[s + 12:s + 24] for s in starts])).clone()                        # (B, T, N, F)
    g = torch.Generator().manual_seed(seed + 1)
    Y[torch.rand(Y.shape, generator=g) < 0.1] = 0.0                                                         # missing readings
    h, outs = None, []
    for t in range(12):
        h = m.tgnn(X[..., t], ei_t, ew_t, h)
        outs.append(m.linear(torch.relu(h)).unsqueeze(1))
    out = torch.cat(outs, dim=1)                                                                            # (B, T, N, 2)
    loss = masked_mae(out, Y)
    loss.backward()
    save(name, edge_index=ei_t, edge_weight=ew_t, X=X, Y=Y, state=sd(m), out=out.detach(), loss=loss.detach(),
         grads={k: p.grad.detach().clone() for k, p in m.named_parameters()})


def tgcn2_seq_metr_la_grads():
    ei, ew, series = synthetic.metr_la_like(0, 256)
    _seq("tgcn2_seq_metr_la_grads", ei, ew, series, 8, 11)


def tgcn2_seq_pems_bay_grads():
    ei, ew, series = synthetic.pems_bay_like(0, 128)
    _seq("tgcn2_seq_pems_bay_grads", ei, ew, series, 4, 12)


def tgcn_chickenpox_seq_grads():
    tg = refload.load("nn.recurrent.temporalgcn")
    z = np.load(os.path.join(ROOT, "pytorch_geometric_temporal_b200", "dataset", "data", "chickenpox.npz"))
    ei = torch.tensor(z["edges"], dtype=torch.int64).T.contiguous()
    ew = torch.ones(ei.shape[1], dtype=torch.float32)
    FX = np.asarray(z["FX"], dtype=np.float32)
    X = torch.from_numpy(np.stack([FX[i:i + 4].T for i in range(24)]).copy())       # (24, 20, 4): snapshot i's features
    Y = torch.from_numpy(np.stack([FX[i + 4] for i in range(24)]).copy())           # (24, 20)
    torch.manual_seed(13)
    m = _Seq(tg.TGCN(4, 32), 32, 1)
    _nonzero_biases(m, 13)
    g = torch.Generator().manual_seed(14)
    H0 = (torch.randn(20, 32, generator=g) * 0.5).requires_grad_(True)
    h, cost, outs = H0, 0, []
    for t in range(24):
        h = m.tgnn(X[t], ei, ew, h)
        y = m.linear(torch.relu(h))
        outs.append(y)
        cost = cost + torch.mean((y - Y[t]) ** 2)        # (20, 1) - (20,) broadcasts, as in the example's cost
    cost = cost / 24
    cost.backward()
    save("tgcn_chickenpox_seq_grads", edge_index=ei, edge_weight=ew, X=X, Y=Y, H0=H0.detach(), state=sd(m),
         out=torch.stack([o.detach() for o in outs]), loss=cost.detach(), gH0=H0.grad.clone(),
         grads={k: p.grad.detach().clone() for k, p in m.named_parameters()})


GENERATORS = {"tgcn2_seq_metr_la_grads": tgcn2_seq_metr_la_grads, "tgcn2_seq_pems_bay_grads": tgcn2_seq_pems_bay_grads,
              "tgcn_chickenpox_seq_grads": tgcn_chickenpox_seq_grads}


if __name__ == "__main__":
    names = sys.argv[1:] or list(GENERATORS)
    for n in names:
        GENERATORS[n]()
