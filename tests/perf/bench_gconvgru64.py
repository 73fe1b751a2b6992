"""GConvGRU at 64 hidden channels on the 64-wide row-split cell kernels (`fused`) against the op-for-op path (`autograd`:
fused_training = False, and for `no_grad` calls the row-split route switched off): the reference's WikiMaths tutorial step at 64 channels
-- GConvGRU(14, 64, 2) + ReLU + Linear(64, 1), H = None, forward, MSE, backward, Adam(lr = 0.01) -- eagerly and replayed from a CUDA
graph; a `no_grad` cell on WikiMaths; and one epoch of the chickenpox example with GConvGRU(4, 64, 2) (H = None per snapshot, cumulative
MSE, one backward, one Adam step).  Configurations alternate within the run, `--runs` times each; every timed run prints one JSON line:
ms per call, the card, its power limit and maximum SM clock (read in the same run) and the library launches per eager call."""
import argparse
import json
import os
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=200, help="timed calls per run (epochs: a tenth of it)")
ap.add_argument("--runs", type=int, default=3)
args = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_gconvgru_wikimaths import capture, card, launches, timed  # noqa: E402
from gconvgru64_seq import RecurrentGCN64  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from wikimaths_seq import load  # noqa: E402

DEV = "cuda"


def _model(F, fused):
    torch.manual_seed(1)
    m = RecurrentGCN64(F, 2).to(DEV)
    m.recurrent.fused_training = fused
    if not fused:
        m.recurrent._rows_ok = lambda *a, **k: False
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    return m, torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)


def wikimaths(fused, graph):
    ei, ew = graph
    m, opt = _model(14, fused)
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
    return {"wikimaths_step": dict(eager=step, graph=capture(step), launches=launches(step)),
            "wikimaths_no_grad": dict(eager=infer, graph=capture(infer), launches=launches(infer))}


def chickenpox(fused):
    ei, ew, X, Y = chickenpox_train_split()
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV)
    m, opt = _model(4, fused)

    def epoch():
        cost = 0
        for t in range(X.size(0)):
            cost = cost + torch.mean((m.linear(torch.relu(m.recurrent(X[t], ei, ew))) - Y[t]) ** 2)
        (cost / X.size(0)).backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
    return {"chickenpox_epoch": dict(eager=epoch, launches=launches(epoch))}


def main():
    g = load(os.path.join(ROOT, "tests", "golden"))
    graph = (g["edge_index"].to(DEV), g["edge_weight"].to(DEV))
    name, pl, clk = card()
    cfgs = {f: {**wikimaths(f == "fused", graph), **chickenpox(f == "fused")} for f in ("fused", "autograd")}
    for run in range(args.runs):
        for what in ("wikimaths_step", "wikimaths_no_grad", "chickenpox_epoch"):
            for f in ("fused", "autograd"):
                c = cfgs[f][what]
                n = max(1, args.steps // 10) if what == "chickenpox_epoch" else args.steps
                for mode in ("eager", "graph"):
                    if mode not in c:
                        continue
                    c[mode]()
                    ms = timed(c[mode], n)
                    print(json.dumps(dict(what=what, path=f, mode=mode, run=run, ms=round(ms, 4), launches=c["launches"], gpu=name,
                                          power_limit_w=pl, max_sm_clock_mhz=clk)), flush=True)


if __name__ == "__main__":
    main()
