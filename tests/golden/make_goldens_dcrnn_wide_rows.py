"""Golden vectors for BatchedDCRNN at 64 hidden channels, the DCRNN paper's width, from the UNMODIFIED reference modules (same mechanism
as make_goldens_dcrnn_rows.py: the reference imported through oracle/refload.py on top of oracle/stubs).  Run in the build container only:
python tests/golden/make_goldens_dcrnn_wide_rows.py

* dcrnn_wide_rows_metr_la.pt.gz  -- BatchedDCRNN(2, 64, 3) on the METR-LA-shaped graph (207 nodes)
* dcrnn_wide_rows_pems_bay.pt.gz -- BatchedDCRNN(2, 64, 2) on the PEMS-BAY-shaped graph (325 nodes)

Each: 2 windows of 12 steps, the reference evaluated in float64 (see `make`), every parameter (nonzero biases included) drawn from a seeded generator by `params()`, so the tests regenerate
the state, the graph and X instead of reading them; stored are gX and the gradient of every parameter of sum(out * linspace(-1, 1)), and
the output at steps OUT_STEPS -- step 0 (the zero-state launch), step 1 (the first full-chain step) and the last.  The gradients depend on
every step's output, so they cover the steps not stored.
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
CASES = {"metr_la": (synthetic.metr_la_like, 3, (7, 40)), "pems_bay": (synthetic.pems_bay_like, 2, (4, 33))}


def params(named_shapes, seed):
    """{name: tensor}: weights uniform in +-1/sqrt(fan) as the reference's glorot scale, biases N(0, 0.1^2), from one generator"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in named_shapes:
        if name.endswith(".bias"):
            out[name] = torch.randn(shape, generator=g) * 0.1
        else:
            a = (6.0 / (shape[-2] + shape[-1])) ** 0.5
            out[name] = (torch.rand(shape, generator=g) * 2 - 1) * a
    return out


def inputs(name):
    """(edge_index, edge_weight, X (2, 12, N, 2), K) of a case"""
    like, K, starts = CASES[name]
    ei, ew, series = like(0, 64)
    X = torch.from_numpy(np.stack([series[s:s + 12] for s in starts]).astype(np.float32))
    return torch.as_tensor(ei), torch.as_tensor(ew, dtype=torch.float32), X, K


def make(name):
    """The reference runs in float64 on the float32 inputs and parameters, and the results are stored in float32: at 64 channels and 12
    steps a float32 run of the reference differs from the exact result by about 1e-5, as much as the kernels' own error, so the golden
    holds the exact values and the test measures the kernels' error alone."""
    dc = refload.load("nn.recurrent.dcrnn")
    ei, ew, X, K = inputs(name)
    state = params([(n_, p.shape) for n_, p in dc.BatchedDCRNN(2, 64, K).named_parameters()], 11)   # drawn in float32, as the tests do
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        m = dc.BatchedDCRNN(2, 64, K)
        with torch.no_grad():
            for k, v in state.items():
                dict(m.named_parameters())[k].copy_(v.double())
        X = X.double().requires_grad_(True)
        out = m(X, ei, ew.double())
        w = torch.linspace(-1, 1, out.numel()).view_as(out)
        (out * w).sum().backward()
    finally:
        torch.set_default_dtype(old)
    path = os.path.join(OUT, f"dcrnn_wide_rows_{name}.pt.gz")
    with gzip.open(path, "wb", compresslevel=9) as f:
        torch.save(dict(out_steps=OUT_STEPS, out=out.detach()[:, OUT_STEPS].float(), gX=X.grad.float(),
                        grads={k: p.grad.detach().float() for k, p in m.named_parameters()}), f)
    print(f"dcrnn_wide_rows_{name}.pt.gz  {os.path.getsize(path) / 1024:.0f} KB")


if __name__ == "__main__":
    for name in CASES:
        make(name)
