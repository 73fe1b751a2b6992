"""Golden vectors for GConvGRU training from the UNMODIFIED reference module (imported through oracle/refload.py on top of oracle/stubs, as
make_goldens_tgcn.py does).  Run in the build container only:   python tests/golden/make_goldens_gconvgru.py [name ...]

The training loop is written here, not copied from the example script (tests/gconvgru_seq.py runs the same loop on this package):
* gconvgru_chickenpox_K{1,2}_{sym,rw}   -- examples/recurrent/gconvgru_example.py's epoch: RecurrentGCN (GConvGRU(4, 32, K), ReLU,
                                           Linear(32, 1)) called once per snapshot of the 20 % train split of chickenpox with H = None,
                                           cumulative MSE divided by the number of snapshots; `rw` with lambda_max = 1.8
* gconvgru_chickenpox_K{1,2}_carried    -- the same snapshots with the state carried from a leaf H0 (dL/dH0 stored)
* gconvgru_metr_la_K2                   -- GConvGRU(2, 32, 2) on the 207-node METR-LA-shaped graph, 12 steps carried from H0
Every file holds every step's prediction, the cost and the gradient of every parameter; biases are set to non-zero values.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import refload  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402


def save(name, **kw):
    torch.save(kw, os.path.join(HERE, name + ".pt"))
    print(f"{name}.pt  {os.path.getsize(os.path.join(HERE, name + '.pt')) / 1024:.0f} KB")


class _Ref(torch.nn.Module):
    def __init__(self, cls, F, K, normalization):
        super().__init__()
        self.recurrent = cls(F, 32, K, normalization=normalization)
        self.linear = torch.nn.Linear(32, 1)


def _case(name, ei, ew, X, Y, K, normalization="sym", lambda_max=None, carried=False, seed=0):
    gru = refload.load("nn.recurrent.gconv_gru")
    torch.manual_seed(seed)
    m = _Ref(gru.GConvGRU, X.shape[-1], K, normalization)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    lam = None if lambda_max is None else torch.tensor(lambda_max)
    H0 = (torch.randn(X.shape[1], 32, generator=g) * 0.5).requires_grad_(True) if carried else None
    h, cost, outs = H0, 0, []
    for t in range(X.shape[0]):
        if carried:
            h = hh = m.recurrent(X[t], ei, ew, h, lambda_max=lam)
        else:
            hh = m.recurrent(X[t], ei, ew, lambda_max=lam)
        y = m.linear(torch.relu(hh))
        outs.append(y)
        cost = cost + torch.mean((y - Y[t]) ** 2)
    cost = cost / X.shape[0]
    cost.backward()
    extra = dict(H0=H0.detach(), gH0=H0.grad.clone()) if carried else {}
    save(name, edge_index=ei, edge_weight=ew, X=X, Y=Y, K=K, normalization=normalization, lambda_max=lam,
         state={k: v.detach().clone() for k, v in m.state_dict().items()}, out=torch.stack([o.detach() for o in outs]),
         loss=cost.detach(), grads={k: p.grad.detach().clone() for k, p in m.named_parameters()}, **extra)


def _chickenpox(K, normalization, lambda_max=None, carried=False):
    ei, ew, X, Y = chickenpox_train_split()
    tag = "carried" if carried else normalization
    _case(f"gconvgru_chickenpox_K{K}_{tag}", ei, ew, X, Y, K, normalization, lambda_max, carried, seed=20 + K)


def gconvgru_metr_la_K2():
    ei, ew, series = synthetic.metr_la_like(0, 64)
    X = torch.from_numpy(series[3:15].copy())                         # (12, 207, 2)
    Y = torch.from_numpy(series[4:16, :, 0].copy())                   # next step's first feature
    _case("gconvgru_metr_la_K2", torch.from_numpy(ei), torch.from_numpy(ew), X, Y, 2, "sym", None, True, seed=31)


GENERATORS = {f"gconvgru_chickenpox_K{K}_{n}": (lambda K=K, n=n: _chickenpox(K, n, 1.8 if n == "rw" else None))
              for K in (1, 2) for n in ("sym", "rw")}
GENERATORS.update({f"gconvgru_chickenpox_K{K}_carried": (lambda K=K: _chickenpox(K, "sym", carried=True)) for K in (1, 2)})
GENERATORS["gconvgru_metr_la_K2"] = gconvgru_metr_la_K2


if __name__ == "__main__":
    for n in sys.argv[1:] or list(GENERATORS):
        GENERATORS[n]()
