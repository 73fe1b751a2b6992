"""The loops of tests/golden/make_goldens_wikimaths.py on this package's modules, shared by the CPU and GPU tests and by
tests/perf/bench_gconvgru_wikimaths.py: the reference's WikiMaths tutorial model (GConvGRU(14, 32, K), ReLU, Linear(32, 1)) over a few
snapshots -- H = None with one backward per snapshot (the tutorial), or the state carried from a leaf H0 with one backward at the end."""
import gzip
import io
import os

import torch

from gconvgru_seq import RecurrentGCN


def carried_h0(n):
    """H0 of the carried case: exact multiples of 1/16 in [-0.5, 0.5], computed rather than stored."""
    i = torch.arange(n).unsqueeze(1) * 7 + torch.arange(32).unsqueeze(0) * 13
    return ((i % 17) - 8).float() / 16


def load(golden_dir):
    """The fixture with the graph as int64 / float32 and the tutorial's windows rebuilt from the stored series:
    X[t] = series[t:t+lags].T (N, lags), Y[t] = series[t+lags] (N,); the carried case's H0 from carried_h0."""
    with gzip.open(os.path.join(golden_dir, "gconvgru_wikimaths.pt.gz"), "rb") as f:
        g = torch.load(io.BytesIO(f.read()), weights_only=False)
    s, lags = g["series"], g["lags"]
    n = s.shape[0] - lags
    g["edge_index"], g["edge_weight"] = g["edge_index"].long(), g["edge_weight"].float()
    g["X"] = torch.stack([s[i:i + lags].T for i in range(n)]).contiguous()
    g["Y"] = torch.stack([s[i + lags] for i in range(n)])
    for c in g["cases"].values():
        if "gH0" in c:
            c["H0"] = carried_h0(s.shape[1])
    return g


def model_for(c, device="cpu", fused=True):
    m = RecurrentGCN(14, c["K"], c["normalization"])
    m.load_state_dict(c["state"])
    m.recurrent.fused_training = fused
    return m.to(device)


def run(m, g, c, device="cpu", H0=None, backward=True):
    """(predictions (S, N, 1), per-snapshot costs (S,)).  H0 None: every snapshot from H = None and, with `backward`, its own backward;
    else the state is carried from H0 and the mean cost is backpropagated once."""
    ei, ew = g["edge_index"].to(device).long(), g["edge_weight"].to(device)
    X, Y = g["X"].to(device), g["Y"].to(device)
    lam = c.get("lambda_max")
    lam = None if lam is None else lam.to(device)
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
