"""Golden vectors for GConvGRU on the reference's WikiMaths data, from the UNMODIFIED reference module (imported through oracle/refload.py,
as make_goldens_gconvgru.py does).  Run in the build container only:   python tests/golden/make_goldens_wikimaths.py

The model is the reference's second tutorial (docs/source/notes/introduction.rst, "Web Traffic Prediction"): GConvGRU(14, 32, K), ReLU,
Linear(32, 1), one snapshot per call.  The data is the reference checkout's dataset/wikivital_mathematics.json (1068 nodes, 27 079
weighted directed edges); the loader's per-node standardisation and 14-lag windows are restated here:
    y = (Y - mean_t Y) / std_t Y  (population std),  x_i = y[i:i+14].T,  target_i = y[i+14]
The fixture is one gzip-compressed torch file: the graph (edge_index int16, the integer link counts as uint8 -- both exact), the
standardised series of the first SNAPSHOTS + 14 periods (the windows are rebuilt from it by tests/wikimaths_seq.py) and these cases, each
with every prediction, the cost and the gradient of every parameter (biases set to non-zero values):
* K2_sym          the tutorial's pattern: H = None, cost_t = mean((y_hat.squeeze() - y_t)^2), one backward per snapshot, parameters fixed
                  (gradients accumulate over the snapshots; no optimiser step)
* K1_sym          the same with K = 1
* K2_sym_carried  H carried from a leaf H0 over the snapshots, cost = mean over snapshots, one backward; plus dL/dH0 (H0 is
                  tests/wikimaths_seq.py's carried_h0, computed, not stored)
The three K = 2 cases start from the same parameters, stored once.
* K2_rw           the tutorial's pattern with normalization = "rw" and lambda_max = 1.6
"""
import gzip
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import refload  # noqa: E402
from wikimaths_seq import carried_h0  # noqa: E402

SNAPSHOTS, LAGS = 6, 14
OUT = os.path.join(HERE, "gconvgru_wikimaths.pt.gz")
_STATES = {}


def wikimaths():
    with open(os.path.join(refload.REFERENCE_ROOT, "dataset", "wikivital_mathematics.json")) as f:
        d = json.load(f)
    ei = np.array(d["edges"]).T
    ew = np.array(d["weights"]).T
    Y = np.stack([np.array(d[str(t)]["y"]) for t in range(d["time_periods"])])
    Y = (Y - Y.mean(axis=0)) / Y.std(axis=0)
    series = torch.from_numpy(Y[:SNAPSHOTS + LAGS].astype(np.float32))
    X = torch.stack([series[i:i + LAGS].T for i in range(SNAPSHOTS)])
    T = torch.stack([series[i + LAGS] for i in range(SNAPSHOTS)])
    return torch.from_numpy(ei.astype(np.int64)), torch.from_numpy(ew.astype(np.float32)), series, X, T


class _Ref(torch.nn.Module):
    def __init__(self, cls, K, normalization):
        super().__init__()
        self.recurrent = cls(LAGS, 32, K, normalization=normalization)
        self.linear = torch.nn.Linear(32, 1)


def case(ei, ew, X, Y, K, normalization="sym", lambda_max=None, carried=False, seed=0):
    gru = refload.load("nn.recurrent.gconv_gru")
    torch.manual_seed(seed)
    m = _Ref(gru.GConvGRU, K, normalization)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    state = _STATES.setdefault((K, seed), {k: v.detach().clone() for k, v in m.state_dict().items()})   # one object per (K, seed)
    assert all(torch.equal(v, m.state_dict()[k]) for k, v in state.items())
    lam = None if lambda_max is None else torch.tensor(lambda_max)
    H0 = carried_h0(X.shape[1]).requires_grad_(True) if carried else None
    h, total, outs, losses = H0, 0, [], []
    for t in range(X.shape[0]):
        if carried:
            h = hh = m.recurrent(X[t], ei, ew, h, lambda_max=lam)
        else:
            hh = m.recurrent(X[t], ei, ew, lambda_max=lam)
        y = m.linear(torch.relu(hh))
        cost = torch.mean((y.squeeze() - Y[t]) ** 2)
        outs.append(y.detach())
        losses.append(cost.detach())
        if carried:
            total = total + cost
        else:
            cost.backward()
    if carried:
        (total / X.shape[0]).backward()
    c = dict(K=K, normalization=normalization, lambda_max=lam, state=state, out=torch.stack(outs), losses=torch.stack(losses),
             grads={k: p.grad.detach().clone() for k, p in m.named_parameters()})
    if carried:
        c.update(gH0=H0.grad.clone())
    return c


def main():
    ei, ew, series, X, Y = wikimaths()
    assert ei.max() < 2 ** 15 and bool((ew == ew.round()).all()) and ew.max() < 256
    cases = {"K2_sym": case(ei, ew, X, Y, 2, seed=41), "K1_sym": case(ei, ew, X, Y, 1, seed=42),
             "K2_sym_carried": case(ei, ew, X, Y, 2, carried=True, seed=41), "K2_rw": case(ei, ew, X, Y, 2, "rw", 1.6, seed=41)}
    buf = io.BytesIO()
    torch.save(dict(edge_index=ei.to(torch.int16), edge_weight=ew.to(torch.uint8), series=series, lags=LAGS, cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
