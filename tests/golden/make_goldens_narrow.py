"""Golden vectors for the narrow-state DCRNN (the model of the reference's index-batching scripts, BatchedDCRNN(F, F, K=3)) from the
UNMODIFIED reference modules (same mechanism as make_goldens_r2.py: the reference imported through oracle/refload.py on top of
oracle/stubs).  Run in the build container only:  python tests/golden/make_goldens_narrow.py [name ...]

Each file stores the output, gX and the gradient of every parameter of sum(out * linspace(-1, 1)):
* dcrnn_narrow_pems_bay -- BatchedDCRNN(2, 2, 3) on the PEMS-BAY-shaped graph (325 nodes), 3 windows of 12 steps
* dcrnn_narrow_metr_la  -- BatchedDCRNN(2, 2, 3) on the METR-LA-shaped graph (207 nodes), 3 windows of 12 steps
* dcrnn_narrow_chickenpox -- BatchedDCRNN(1, 1, 3) on the chickenpox graph (20 nodes, 102 edges with self loops), 5 windows of 4 steps
                             (get_index_dataset's default lags=4, chicken_pox_main.py)
* dcrnn_narrow_cell     -- DCRNN(2, 2, 3) (the non-batched DConv) with an incoming H on the METR-LA-shaped graph: output, gX, gH and the
                           parameter gradients
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
            if n_.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)


def _batched(name, ei, ew, series, starts, horizon, F, seed):
    dc = refload.load("nn.recurrent.dcrnn")
    ei_t, ew_t = torch.as_tensor(ei), torch.as_tensor(ew, dtype=torch.float32)
    torch.manual_seed(seed)
    m = dc.BatchedDCRNN(F, F, 3)
    _nonzero_biases(m, seed)
    X = torch.from_numpy(np.stack([series[s:s + horizon] for s in starts]).astype(np.float32)).clone().requires_grad_(True)
    out = m(X, ei_t, ew_t)
    w = torch.linspace(-1, 1, out.numel()).view_as(out)
    (out * w).sum().backward()
    save(name, edge_index=ei_t, edge_weight=ew_t, X=X.detach(), state=sd(m), out=out.detach(), gX=X.grad.clone(),
         grads={k: p.grad.detach().clone() for k, p in m.named_parameters()}, K=3, F=F)


def dcrnn_narrow_pems_bay():
    ei, ew, series = synthetic.pems_bay_like(0, 64)
    _batched("dcrnn_narrow_pems_bay", ei, ew, series, [2, 19, 40], 12, 2, 0)


def dcrnn_narrow_metr_la():
    ei, ew, series = synthetic.metr_la_like(0, 64)
    _batched("dcrnn_narrow_metr_la", ei, ew, series, [3, 20, 41], 12, 2, 1)


def dcrnn_narrow_chickenpox():
    z = np.load(os.path.join(ROOT, "pytorch_geometric_temporal_b200", "dataset", "data", "chickenpox.npz"))
    ei = torch.tensor(z["edges"], dtype=torch.int64).T.contiguous()
    ew = torch.ones(ei.shape[1], dtype=torch.float32)
    series = np.asarray(z["FX"], dtype=np.float32)[:, :, None]          # (521, 20, 1), as get_index_dataset expands it
    _batched("dcrnn_narrow_chickenpox", ei, ew, series, [0, 7, 100, 250, 510], 4, 1, 2)


def dcrnn_narrow_cell():
    dc = refload.load("nn.recurrent.dcrnn")
    ei, ew, series = synthetic.metr_la_like(0, 16)
    ei_t, ew_t = torch.from_numpy(ei), torch.from_numpy(ew)
    torch.manual_seed(3)
    m = dc.DCRNN(2, 2, 3)
    _nonzero_biases(m, 3)
    g = torch.Generator().manual_seed(4)
    X = torch.from_numpy(series[5].astype(np.float32)).clone().requires_grad_(True)     # (207, 2)
    H = (torch.randn(207, 2, generator=g) * 0.5).requires_grad_(True)
    out = m(X, ei_t, ew_t, H)
    w = torch.linspace(-1, 1, out.numel()).view_as(out)
    (out * w).sum().backward()
    save("dcrnn_narrow_cell", edge_index=ei_t, edge_weight=ew_t, X=X.detach(), H=H.detach(), state=sd(m), out=out.detach(),
         gX=X.grad.clone(), gH=H.grad.clone(), grads={k: p.grad.detach().clone() for k, p in m.named_parameters()}, K=3)


GENERATORS = {"dcrnn_narrow_pems_bay": dcrnn_narrow_pems_bay, "dcrnn_narrow_metr_la": dcrnn_narrow_metr_la,
              "dcrnn_narrow_chickenpox": dcrnn_narrow_chickenpox, "dcrnn_narrow_cell": dcrnn_narrow_cell}


if __name__ == "__main__":
    names = sys.argv[1:] or list(GENERATORS)
    for n in names:
        GENERATORS[n]()
