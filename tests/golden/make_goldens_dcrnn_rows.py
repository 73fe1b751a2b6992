"""Golden vectors for BatchedDCRNN(2, 32, 2) on a graph too large for the one-SM kernels, from the UNMODIFIED reference modules (same
mechanism as make_goldens_narrow.py: the reference imported through oracle/refload.py on top of oracle/stubs).  Run in the build
container only:  python tests/golden/make_goldens_dcrnn_rows.py

* dcrnn_rows_pems_bay.pt.gz -- BatchedDCRNN(2, 32, 2) on the PEMS-BAY-shaped graph (325 nodes, 2694 edges), 2 windows of 12 steps,
                               nonzero biases: gX and the gradient of every parameter of sum(out * linspace(-1, 1)), and the output at
                               steps OUT_STEPS -- step 0 (the zero-state launch), step 1 (the first two-launch step) and the last.  The
                               gradients depend on every step's output, so they cover the steps not stored; storing the whole output
                               would double the fixture.
"""
import gzip
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refload  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
OUT_STEPS = [0, 1, 11]


def dcrnn_rows_pems_bay():
    dc = refload.load("nn.recurrent.dcrnn")
    ei, ew, series = synthetic.pems_bay_like(0, 64)
    ei_t, ew_t = torch.as_tensor(ei), torch.as_tensor(ew, dtype=torch.float32)
    torch.manual_seed(5)
    m = dc.BatchedDCRNN(2, 32, 2)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    X = torch.from_numpy(np.stack([series[s:s + 12] for s in (4, 33)]).astype(np.float32)).clone().requires_grad_(True)
    out = m(X, ei_t, ew_t)
    w = torch.linspace(-1, 1, out.numel()).view_as(out)
    (out * w).sum().backward()
    path = os.path.join(OUT, "dcrnn_rows_pems_bay.pt.gz")
    with gzip.open(path, "wb", compresslevel=9) as f:
        torch.save(dict(edge_index=ei_t.to(torch.int32), edge_weight=ew_t, X=X.detach(),
                        state={k: v.detach().clone() for k, v in m.state_dict().items()}, out_steps=OUT_STEPS,
                        out=out.detach()[:, OUT_STEPS].clone(), gX=X.grad.clone(),
                        grads={k: p.grad.detach().clone() for k, p in m.named_parameters()}), f)
    print(f"dcrnn_rows_pems_bay.pt.gz  {os.path.getsize(path) / 1024:.0f} KB")


if __name__ == "__main__":
    dcrnn_rows_pems_bay()
