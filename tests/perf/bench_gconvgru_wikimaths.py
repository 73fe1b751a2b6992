"""The reference's WikiMaths tutorial step (docs/source/notes/introduction.rst, "Web Traffic Prediction"): RecurrentGCN = GConvGRU(14, 32, 2)
+ ReLU + Linear(32, 1) on the 1068-node, 27 079-edge WikiMaths graph (tests/golden/gconvgru_wikimaths.pt.gz) with seeded features of the
tutorial's shape, H = None at every call; one step = forward, MSE, backward and one Adam(lr = 0.01) step.  Times that step and a `no_grad`
call on the row-split cell kernels (`fused`) and on the op-for-op autograd path (`autograd`), each eagerly and replayed from a CUDA graph.
A last pair of lines times one cell on the chickenpox graph (20 nodes) on the row-split kernels against the one-SM kernel
(stmp_gru_seq_fwd), at the ops level.  Configurations alternate within the run, `--runs` times each; every timed run prints one JSON
line: ms per call, the card and its power limit and maximum SM clock (read in the same run), and the library launches per eager call."""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=200, help="timed calls per run")
ap.add_argument("--runs", type=int, default=3)
args = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from pytorch_geometric_temporal_b200 import _lib, ops  # noqa: E402
from pytorch_geometric_temporal_b200.plan import GraphPlan  # noqa: E402
from gconvgru_seq import RecurrentGCN, chickenpox_train_split  # noqa: E402
from wikimaths_seq import load  # noqa: E402

DEV = "cuda"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        pl, clk = float(q[0]), float(q[1])
    except (OSError, subprocess.SubprocessError, ValueError, IndexError):
        pl = clk = None
    return torch.cuda.get_device_name(), pl, clk


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def capture(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def tutorial(fused, graph):
    ei, ew = graph
    torch.manual_seed(1)
    m = RecurrentGCN(14, 2).to(DEV)
    if not fused:                        # every call, training or not, on the op-for-op path
        m.recurrent._rows_ok = lambda *a, **k: False
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    x = torch.randn(ei.max().item() + 1, 14, device=DEV)
    y = torch.randn(x.size(0), device=DEV)

    def step():
        cost = torch.mean((m.linear(torch.relu(m.recurrent(x, ei, ew))).squeeze() - y) ** 2)
        cost.backward()
        opt.step()
        opt.zero_grad(set_to_none=False)

    def infer():
        with torch.no_grad():
            m.recurrent(x, ei, ew)
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    out = {}
    for name, fn in (("train_step", step), ("no_grad", infer)):
        out[name] = dict(eager=fn, graph=capture(fn), launches=launches(fn))
    return out


def chickenpox_cells():
    ei, ew, X, _ = chickenpox_train_split()
    plan = GraphPlan(_lib.FLAVOR_CHEB, ei.to(DEV), ew.to(DEV), 20, "sym")
    torch.manual_seed(2)
    wcat = torch.zeros(96, 112, device=DEV)
    wcat[:, :64] = torch.randn(96, 64, device=DEV) * 0.15
    wcat[:, 96:100] = torch.randn(96, 4, device=DEV) * 0.3
    wcat[:, 100:104] = torch.randn(96, 4, device=DEV) * 0.3
    bcat = torch.randn(96, device=DEV) * 0.1
    cols = [96 + 4 * (m // 36) + m % 36 if m % 36 < 4 else 32 * (m // 36) + m % 36 - 4 for m in range(72)]
    wr = wcat[:, cols].contiguous()
    img = ops.gru_weight_image(wcat, bcat)
    x, h = X[0].to(DEV), torch.randn(20, 32, device=DEV) * 0.5
    x4, h3 = x.view(1, 1, 20, 4), h.view(1, 20, 32)
    one_sm = lambda: ops.gru_seq_fwd(plan, 1, x4, wcat, bcat, h0=h3, wimage=img)          # noqa: E731
    rows = lambda: ops.gru_rows_fwd(plan, 1, x, h, wr, bcat)                               # noqa: E731
    return {"one_sm": dict(eager=one_sm, graph=capture(one_sm), launches=launches(one_sm)),
            "row_split": dict(eager=rows, graph=capture(rows), launches=launches(rows))}


def main():
    gpu, plimit, clk = card()
    g = load(os.path.join(ROOT, "tests", "golden"))
    graph = (g["edge_index"].to(DEV).long(), g["edge_weight"].to(DEV))
    cfgs = {("wikimaths", fused): tutorial(fused, graph) for fused in (True, False)}
    cells = chickenpox_cells()
    for r in range(args.runs):
        for mode in ("eager", "graph"):
            for what in ("train_step", "no_grad"):
                for (_, fused), c in cfgs.items():
                    ms = timed(c[what][mode], args.steps)
                    print(json.dumps({"bench": "gconvgru_wikimaths", "call": what, "path": "fused" if fused else "autograd", "mode": mode,
                                      "run": r, "ms_per_call": round(ms, 4), "library_launches_per_call": c[what]["launches"], "gpu": gpu,
                                      "power_limit_w": plimit, "max_sm_clock_mhz": clk}), flush=True)
            for name, c in cells.items():
                ms = timed(c[mode], args.steps)
                print(json.dumps({"bench": "gconvgru_cell_chickenpox", "call": "no_grad H given, K = 2, cin = 4", "path": name, "mode": mode,
                                  "run": r, "ms_per_call": round(ms, 4), "library_launches_per_call": c["launches"], "gpu": gpu,
                                  "power_limit_w": plimit, "max_sm_clock_mhz": clk}), flush=True)


if __name__ == "__main__":
    main()
