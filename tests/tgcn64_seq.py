"""The TGCN / A3TGCN cases of tests/golden/make_goldens_tgcn64.py at 64 hidden channels, shared by that generator, the GPU tests of the
64-wide fused kernels and tests/perf/bench_tgcn64.py:
* tgcn2_metr_la, tgcn2_pems_bay -- BatchedTGCN: TGCN2(2, 64, 1) + ReLU + Linear(64, 2) over 12 steps, H = None at t = 0 and then carried,
                                   2 windows of the METR-LA- / PEMS-BAY-shaped series laid out (B, N, F, T), masked MAE with some zero targets
* tgcn_chickenpox               -- TGCN(4, 64) + ReLU + Linear(64, 1) over the first 24 chickenpox snapshots from a leaf state H0,
                                   cumulative MSE / 24; also dL/dH0
* a3tgcn2_cfg3                  -- the A3TGCN2(2, 64, 12) training call at the PEMS-BAY shape (325 nodes, 4 rows, H = None), loss
                                   sum(out * wgt) / numel
* a3tgcn_shared_h               -- an A3TGCN(4, 64, 4) inference call on the chickenpox graph with one state H for every period
The fixture stays small (lstm64_seq.py's scheme): a case's parameters come from its seed (`seeded_state`) and its inputs from the in-tree
synthetic series and chickenpox data, and the reference's float64 results are stored as fingerprints next to its exact loss.  A test runs
the in-tree float64 oracle on the case, checks it against the fingerprints (`check_reference`), then holds the module to the oracle."""
import gzip
import io
import os

import numpy as np
import torch

from lstm64_seq import fingerprint
from oracle import recurrent as R
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN, A3TGCN2, TGCN, TGCN2

WIDTH = 64
FIXTURE = "tgcn64.pt.gz"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = {
    "tgcn2_metr_la": dict(kind="seq", graph="metr_la", seed=21),
    "tgcn2_pems_bay": dict(kind="seq", graph="pems_bay", seed=22),
    "tgcn_chickenpox": dict(kind="chickenpox", seed=23),
    "a3tgcn2_cfg3": dict(kind="a3_train", seed=24),
    "a3tgcn_shared_h": dict(kind="a3_shared", seed=25),
}


class SeqModel(torch.nn.Module):
    """The model of a case (state_dict keys tgnn.*, linear.*); `mods` holds the TGCN / TGCN2 / A3TGCN / A3TGCN2 classes to build from (this
    package's or the reference's)."""

    def __init__(self, c, mods):
        super().__init__()
        if c["kind"] == "seq":
            self.tgnn, self.linear = mods["TGCN2"](2, WIDTH, 1), torch.nn.Linear(WIDTH, 2)
        elif c["kind"] == "chickenpox":
            self.tgnn, self.linear = mods["TGCN"](4, WIDTH), torch.nn.Linear(WIDTH, 1)
        elif c["kind"] == "a3_train":
            self.tgnn = mods["A3TGCN2"](2, WIDTH, 12, 4)
        else:
            self.tgnn = mods["A3TGCN"](4, WIDTH, 4)


MODS = {"TGCN": TGCN, "TGCN2": TGCN2, "A3TGCN": A3TGCN, "A3TGCN2": A3TGCN2}


def seeded_state(c):
    """The parameters of a case from its seed (float32 values): weight matrices N(0, 1/fan_in), everything else N(0, 0.01), in the sorted
    order of the state_dict keys, which this package's modules share with the reference's."""
    keys = SeqModel(c, MODS).state_dict()
    g = torch.Generator().manual_seed(c["seed"])
    state = {}
    for k in sorted(keys):
        shape = keys[k].shape
        scale = shape[-1] ** -0.5 if len(shape) == 2 and min(shape) > 1 else 0.1
        state[k] = (torch.randn(shape, generator=g, dtype=torch.float64) * scale).float()
    return state


def _chickenpox():
    z = np.load(os.path.join(ROOT, "pytorch_geometric_temporal_b200", "dataset", "data", "chickenpox.npz"))
    ei = torch.tensor(z["edges"], dtype=torch.int64).T.contiguous()
    return ei, torch.ones(ei.shape[1], dtype=torch.float32), np.asarray(z["FX"], dtype=np.float32)


def data(c, device="cpu"):
    """The inputs of case c (float32 whatever the default dtype): edge_index, edge_weight and X, plus Y (seq, chickenpox), H0
    (chickenpox), wgt (a3_train) or H (a3_shared)."""
    g = torch.Generator().manual_seed(c["seed"] + 1)
    if c["kind"] == "seq":
        ei, ew, series = (synthetic.metr_la_like if c["graph"] == "metr_la" else synthetic.pems_bay_like)(0, 128)
        starts = [5, 22]
        X = torch.from_numpy(np.stack([series[s:s + 12] for s in starts])).permute(0, 2, 3, 1).contiguous()   # (B, N, F, T)
        Y = torch.from_numpy(np.stack([series[s + 12:s + 24] for s in starts])).clone()                       # (B, T, N, F)
        Y[torch.rand(Y.shape, generator=g, dtype=torch.float32) < 0.1] = 0.0                                  # missing readings
        d = dict(edge_index=torch.from_numpy(ei), edge_weight=torch.from_numpy(ew), X=X, Y=Y)
    elif c["kind"] == "chickenpox":
        ei, ew, FX = _chickenpox()
        X = torch.from_numpy(np.stack([FX[i:i + 4].T for i in range(24)]).copy())          # (24, 20, 4)
        Y = torch.from_numpy(np.stack([FX[i + 4] for i in range(24)]).copy())              # (24, 20)
        d = dict(edge_index=ei, edge_weight=ew, X=X, Y=Y, H0=torch.randn(20, WIDTH, generator=g, dtype=torch.float32) * 0.5)
    elif c["kind"] == "a3_train":
        ei, ew, _ = synthetic.pems_bay_like(0, 16)
        X = torch.randn(4, 325, 2, 12, generator=g, dtype=torch.float32)
        d = dict(edge_index=torch.from_numpy(ei), edge_weight=torch.from_numpy(ew), X=X,
                 wgt=torch.randn(4, 325, WIDTH, generator=g, dtype=torch.float32))
    else:
        ei, ew, FX = _chickenpox()
        X = torch.randn(20, 4, 4, generator=g, dtype=torch.float32)
        d = dict(edge_index=ei, edge_weight=ew, X=X, H=torch.randn(20, WIDTH, generator=g, dtype=torch.float32) * 0.5)
    return {k: v.to(device) for k, v in d.items()}


def load(golden_dir):
    """{case name: case} with the reference's loss and fingerprints (tests/golden/tgcn64.pt.gz) added to CASES."""
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        stored = torch.load(io.BytesIO(f.read()), weights_only=False)
    return {k: {**CASES[k], **stored[k]} for k in CASES}


def model_for(c, device="cpu", fused=True):
    m = SeqModel(c, MODS)
    m.load_state_dict(seeded_state(c))
    base = m.tgnn._base_tgcn if c["kind"].startswith("a3") else m.tgnn
    base.fused_training = fused
    return m.to(device)


def masked_mae(pred, true):
    """The index-batching scripts' masked MAE; NaNs are zeroed with torch.where so that a CUDA graph can capture it."""
    mask = (true != 0).to(pred.dtype)
    mask = mask / mask.mean()
    loss = torch.abs(pred - true) * mask
    return torch.where(loss != loss, torch.zeros_like(loss), loss).mean()


def run(m, c, d, backward=True, leaves=None):
    """{"out", "loss" (None for inference), and after the backward "grads" {name: gradient} [, "gH0"]} of case c on inputs d.  `leaves`
    (name -> tensor) stands for m's parameters when the gradients are taken w.r.t. other tensors (the oracle's)."""
    ei, ew, X = d["edge_index"], d["edge_weight"], d["X"]
    kind = c["kind"]
    res = {"loss": None}
    if kind == "seq":
        h, outs = None, []
        for t in range(X.shape[-1]):
            h = m.tgnn(X[..., t], ei, ew, h)
            outs.append(m.linear(torch.relu(h)).unsqueeze(1))
        res["out"] = torch.cat(outs, dim=1)
        res["loss"] = masked_mae(res["out"], d["Y"].to(res["out"].dtype))
    elif kind == "chickenpox":
        H0 = d["H0"].clone().to(X.dtype if leaves is None else torch.float64).requires_grad_(backward)
        res["H0"] = H0
        h, cost, outs = H0, 0, []
        for t in range(X.shape[0]):
            h = m.tgnn(X[t], ei, ew, h)
            y = m.linear(torch.relu(h))
            outs.append(y)
            cost = cost + torch.mean((y - d["Y"][t].to(y.dtype)) ** 2)      # (20, 1) - (20,) broadcasts, as in the example's cost
        res["out"], res["loss"] = torch.stack(outs), cost / X.shape[0]
    elif kind == "a3_train":
        res["out"] = m.tgnn(X, ei, ew)
        res["loss"] = (res["out"] * d["wgt"].to(res["out"].dtype)).sum() / res["out"].numel()
    else:
        with torch.no_grad():
            res["out"] = m.tgnn(X, ei, ew, d["H"].to(X.dtype))
    if backward and res["loss"] is not None:
        named = dict(m.named_parameters()) if leaves is None else leaves
        extra = [res["H0"]] if "H0" in res else []
        g = torch.autograd.grad(res["loss"], list(named.values()) + extra)
        res["grads"] = dict(zip(named, g[:len(named)]))
        if extra:
            res["gH0"] = g[-1]
    res.pop("H0", None)
    return res


class _Oracle:
    """The in-tree float64 oracle (oracle/recurrent.py) with a module's call signature, on parameter leaves p."""

    def __init__(self, p, a3):
        self.p, self.a3 = p, a3

    def __call__(self, X, ei, ew, H=None):
        f = R.a3tgcn if self.a3 else R.tgcn_cell
        if H is None:
            H = torch.zeros(*X.shape[:(-2 if self.a3 else -1)], WIDTH, dtype=X.dtype, device=X.device)
        return f(self.p, X, ei, ew, H)


def oracle_run(c, d):
    """run() of case c in float64 on the in-tree oracle: (out, loss, {parameter: gradient}, {"gH0": ...} or {})."""
    leaves = {k: v.double().to(d["X"].device).requires_grad_(True) for k, v in seeded_state(c).items()}
    p = {k[len("tgnn."):]: v for k, v in leaves.items() if k.startswith("tgnn.")}
    m = torch.nn.Module()
    m.tgnn = _Oracle(p, c["kind"].startswith("a3"))
    if "linear.weight" in leaves:
        m.linear = lambda t: torch.nn.functional.linear(t, leaves["linear.weight"], leaves["linear.bias"])
    d64 = {k: v.double() if v.is_floating_point() else v for k, v in d.items()}
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        res = run(m, c, d64, leaves=leaves)
    finally:
        torch.set_default_dtype(old)
    return res["out"], res["loss"], res.get("grads", {}), ({"gH0": res["gH0"]} if "gH0" in res else {})


def check_reference(c, out, loss, grads, extra):
    """The float64 oracle's results of case c against the unmodified reference's, stored as fingerprints and an exact loss."""
    if loss is None:
        assert c["loss"] is None
    else:
        assert abs(float(loss.detach()) - float(c["loss"])) <= 1e-10 * abs(float(c["loss"])), (float(loss.detach()), float(c["loss"]))
    got = {"out": out, **{f"grad/{k}": v for k, v in grads.items()}, **extra}
    assert sorted(got) == sorted(c["fingerprints"])
    for k, t in got.items():
        want = c["fingerprints"][k]
        assert torch.allclose(fingerprint(t), want, rtol=0, atol=1e-9 * float(want[-1]) + 1e-300), k
