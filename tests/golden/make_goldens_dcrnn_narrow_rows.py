"""Golden vectors for BatchedDCRNN(2, 2, 3) on a graph too large for the one-SM narrow kernels, from the UNMODIFIED reference modules (same
mechanism as make_goldens_dcrnn_rows.py: the reference imported through oracle/refload.py on top of oracle/stubs).  Run in the build
container only:  python tests/golden/make_goldens_dcrnn_narrow_rows.py

* dcrnn_narrow_rows_banded.pt.gz -- BatchedDCRNN(2, 2, 3), the reference's full-PeMS training model, on synthetic.banded_graph(2000, 16000,
                                    seed 3) plus a ring (every DConv norm finite), 2 windows of 12 steps, nonzero biases: gX and the
                                    gradient of every parameter of sum(out * linspace(-1, 1)), and the output at steps OUT_STEPS -- step 0
                                    (the zero-state launch), step 1 (the first full chain) and the last.  The graph and X are not stored:
                                    `inputs()` regenerates them exactly from their seeds (numpy and the CPU torch generator).
"""
import gzip
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
OUT_STEPS = [0, 1, 11]
N = 2000


def inputs():
    """(edge_index int64 (2, E), edge_weight float32 (E,), X float32 (2, 12, N, 2)) on the CPU, from seeds"""
    ei, ew = synthetic.banded_graph(N, 8 * N, span=32, seed=3)
    ring = np.arange(N)
    ei = np.concatenate([ei, np.stack([ring, (ring + 1) % N])], axis=1)
    ew = np.concatenate([ew, np.full(N, 0.5, dtype=np.float32)])
    X = torch.randn(2, 12, N, 2, generator=torch.Generator().manual_seed(3))
    return torch.from_numpy(ei), torch.from_numpy(ew), X


def dcrnn_narrow_rows_banded():
    from oracle import refload
    dc = refload.load("nn.recurrent.dcrnn")
    ei, ew, X = inputs()
    torch.manual_seed(3)
    m = dc.BatchedDCRNN(2, 2, 3)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    X = X.clone().requires_grad_(True)
    out = m(X, ei, ew)
    w = torch.linspace(-1, 1, out.numel()).view_as(out)
    (out * w).sum().backward()
    path = os.path.join(OUT, "dcrnn_narrow_rows_banded.pt.gz")
    with gzip.open(path, "wb", compresslevel=9) as f:
        torch.save(dict(state={k: v.detach().clone() for k, v in m.state_dict().items()}, out_steps=OUT_STEPS,
                        out=out.detach()[:, OUT_STEPS].clone(), gX=X.grad.clone(),
                        grads={k: p.grad.detach().clone() for k, p in m.named_parameters()}), f)
    print(f"dcrnn_narrow_rows_banded.pt.gz  {os.path.getsize(path) / 1024:.0f} KB")


if __name__ == "__main__":
    dcrnn_narrow_rows_banded()
