"""The LSTM tutorial loop of tests/lstm_seq.py at 64 hidden channels -- GConvLSTM or GCLSTM(F, 64, K), ReLU, Linear(64, 1), H and C
carried from None (or from leaf H0 / C0), a cumulative MSE divided by the number of snapshots and one backward at the end -- on the
WikiMaths fixture of tests/wikimaths_seq.py and on the in-tree chickenpox split, shared by tests/golden/make_goldens_lstm64.py, the CPU and
GPU tests of the 64-wide row-split LSTM cell and tests/perf/bench_lstm64.py.

The fixture stays small: a case's parameters are generated from its seed (`seeded_state`), and the unmodified reference's float64 results
are stored as fingerprints (`fingerprint`: four fixed random projections and the norm of each tensor) next to its exact costs.  A test runs
the in-tree float64 oracle (oracle/recurrent.py) on the same case, checks it against those fingerprints (`check_reference`) and then holds
the module under test to the oracle's tensors element by element."""
import gzip
import io
import os
import types

import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200.nn.recurrent import GCLSTM, GConvLSTM

WIDTH = 64
MODULES = {"gconv_lstm": GConvLSTM, "gc_lstm": GCLSTM}
ORACLE = {"gconv_lstm": R.gconv_lstm_cell, "gc_lstm": R.gc_lstm_cell}
FIXTURE = "lstm64.pt.gz"


class RecurrentGCN64(torch.nn.Module):
    """The examples' model at 64 channels (state_dict keys recurrent.*, linear.*); `cls` is the GConvLSTM or GCLSTM class (this package's
    or the reference's)."""

    def __init__(self, cls, node_features, K, normalization="sym"):
        super().__init__()
        self.recurrent = cls(node_features, WIDTH, K, normalization=normalization)
        self.linear = torch.nn.Linear(WIDTH, 1)


def carried_state(n, a, b, m):
    """A leaf state of exact multiples of 1/16 in [-0.5, 0.5], computed rather than stored."""
    i = torch.arange(n).unsqueeze(1) * a + torch.arange(WIDTH).unsqueeze(0) * b
    return ((i % m) - (m // 2)).float() / 16


def seeded_state(module, F, K, seed):
    """The parameters of a case, from its seed alone (float32 values): weight matrices N(0, 1/fan_in), everything else N(0, 0.01), in the
    sorted order of the state_dict keys, which this package's modules share with the reference's."""
    keys = RecurrentGCN64(MODULES[module], F, K).state_dict()
    g = torch.Generator().manual_seed(seed)
    state = {}
    for k in sorted(keys):
        shape = keys[k].shape
        scale = shape[-1] ** -0.5 if len(shape) == 2 and min(shape) > 1 else 0.1
        state[k] = (torch.randn(shape, generator=g, dtype=torch.float64) * scale).float()
    return state


def fingerprint(t):
    """float64 [4 projections onto fixed N(0, 1) vectors, norm] of a tensor: two float64 computations of the same quantity agree to far
    below 1e-9 of the norm, while a wrong element moves them by its error times O(1)."""
    t = t.detach().double().flatten().cpu()
    V = torch.randn(t.numel(), 4, generator=torch.Generator().manual_seed(t.numel()), dtype=torch.float64)
    return torch.cat([t @ V, t.norm().view(1)])


def load(golden_dir):
    """The 64-wide cases (tests/golden/lstm64.pt.gz): each case's module, F, K, normalization, lambda_max and seed, the reference's cost
    and the fingerprints of its predictions and gradients."""
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        return torch.load(io.BytesIO(f.read()), weights_only=False)


def model_for(c, device="cpu", fused=True):
    m = RecurrentGCN64(MODULES[c["module"]], c["F"], c["K"], c["normalization"])
    m.load_state_dict(seeded_state(c["module"], c["F"], c["K"], c["seed"]))
    m.recurrent.fused_training = fused
    return m.to(device)


def oracle_run(c, X, Y, ei, ew, lam=None, H0=None, C0=None):
    """run() of case c in float64 on the in-tree oracle cell: (outs, cost, {parameter name: leaf}); H0 / C0, when given, are float64 leaves
    that require grad."""
    leaves = {k: v.double().to(X.device).requires_grad_(True) for k, v in seeded_state(c["module"], c["F"], c["K"], c["seed"]).items()}
    p = {k[len("recurrent."):]: v for k, v in leaves.items() if k.startswith("recurrent.")}
    cell, norm = ORACLE[c["module"]], c["normalization"]

    def recurrent(x, ei_, ew_, h, cc, lambda_max=None):
        zeros = torch.zeros(x.size(0), WIDTH, dtype=torch.float64, device=x.device)
        return cell(p, x, ei_, ew_, zeros if h is None else h, zeros if cc is None else cc, lambda_max=lambda_max, normalization=norm)
    m = types.SimpleNamespace(recurrent=recurrent,
                              linear=lambda t: torch.nn.functional.linear(t, leaves["linear.weight"], leaves["linear.bias"]))
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        outs, cost = run(m, X.double(), Y.double(), ei, ew.double(), None if lam is None else lam.double(), H0, C0)
    finally:
        torch.set_default_dtype(old)
    return outs, cost, leaves


def check_reference(c, outs, cost, grads, gH0=None, gC0=None):
    """The float64 oracle's results of case c against the unmodified reference's, stored as fingerprints and an exact cost."""
    cost = float(cost.detach())
    assert abs(cost - float(c["cost"])) <= 1e-10 * abs(float(c["cost"])), (cost, float(c["cost"]))
    got = {"out": outs, **{f"grad/{k}": v for k, v in grads.items()}}
    if gH0 is not None:
        got.update({"gH0": gH0, "gC0": gC0})
    assert sorted(got) == sorted(c["fingerprints"])
    for k, t in got.items():
        want = c["fingerprints"][k]
        assert torch.allclose(fingerprint(t), want, rtol=0, atol=1e-9 * float(want[-1]) + 1e-300), k


def run(m, X, Y, ei, ew, lam=None, H0=None, C0=None):
    """(every step's prediction (S, N, 1), cost): H and C carried from H0 / C0 (None: the module's zeros), cumulative MSE / S."""
    h, c, cost, outs = H0, C0, 0, []
    for t in range(X.shape[0]):
        h, c = m.recurrent(X[t], ei, ew, h, c, lambda_max=lam)
        y = m.linear(torch.relu(h))
        outs.append(y)
        cost = cost + torch.mean((y - Y[t]) ** 2)      # (N, 1) - (N,) broadcasts, as in the examples' cost
    return torch.stack(outs), cost / X.shape[0]
