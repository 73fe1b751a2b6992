"""GConvLSTM and GCLSTM at 64 hidden channels on the 64-wide row-split LSTM cell (`rows`) against the routes they replace:
* the WikiMaths tutorial step -- (14, 64, 2) + ReLU + Linear(64, 1), H and C carried from None within the step, MSE, backward,
  Adam(lr = 0.01) -- eagerly and replayed from a CUDA graph, against fused_training = False (`autograd`, op for op);
* a `no_grad` cell (H and C given) against the SpMM + wgmma route (`gemm_lstm`) at in_channels 4 and 16, and against the op-for-op
  inference path at 14, on WikiMaths (1 068 nodes), on random graphs of 2 000 to 32 000 nodes (where ops.LSTM_WIDE_ROWS_GEMM_NODES is
  chosen) and at 50 000 nodes;
* one epoch of the chickenpox example with (4, 64, 2) (H and C carried, cumulative MSE, one backward, one Adam step).
Configurations alternate within the run, `--runs` times each; every timed run prints one JSON line: ms per call, the card, its power limit
and maximum SM clock (read in the same run) and the library launches per eager call."""
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
from pytorch_geometric_temporal_b200 import ops  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from lstm64_seq import MODULES, RecurrentGCN64  # noqa: E402
from wikimaths_seq import load  # noqa: E402

DEV = "cuda"
NO_GRAD_SIZES = (2000, 4000, 8000, 16000, 32000, 50000)


def _model(name, F, fused):
    torch.manual_seed(1)
    m = RecurrentGCN64(MODULES[name], F, 2).to(DEV)
    m.recurrent.fused_training = fused
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    return m, torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)


def _random_graph(n, deg=8):
    g = torch.Generator().manual_seed(n)
    src, dst = torch.randint(0, n, (deg * n,), generator=g), torch.randint(0, n, (deg * n,), generator=g)
    keep = src != dst
    ei = torch.unique(torch.stack([src[keep], dst[keep]]), dim=1)
    return ei.to(DEV), (torch.rand(ei.size(1), generator=g) + 0.1).to(DEV)


def wikimaths_step(name, fused, graph):
    ei, ew = graph
    m, opt = _model(name, 14, fused)
    x = torch.randn(ei.max().item() + 1, 14, device=DEV)
    y = torch.randn(x.size(0), device=DEV)

    def step():
        h, c = m.recurrent(x, ei, ew)
        cost = torch.mean((m.linear(torch.relu(h)).squeeze() - y) ** 2)
        cost.backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
    return dict(eager=step, graph=capture(step), launches=launches(step))


def no_grad_cell(name, cin, graph, path):
    """`rows`: the 64-wide cell whatever the node count; `gemm_lstm`: the SpMM + wgmma route (cin % 4 == 0); `op_for_op`: neither."""
    ei, ew = graph
    n = ei.max().item() + 1
    torch.manual_seed(2)
    m = MODULES[name](cin, 64, 2).to(DEV)
    x, h, c = torch.randn(n, cin, device=DEV), torch.randn(n, 64, device=DEV), torch.randn(n, 64, device=DEV)
    limit = {"rows": 1 << 62, "gemm_lstm": 0, "op_for_op": 0}[path]
    if path == "op_for_op":
        m._rows_ok = lambda *a, **k: False

    def infer():
        saved, ops.LSTM_WIDE_ROWS_GEMM_NODES = ops.LSTM_WIDE_ROWS_GEMM_NODES, limit
        try:
            with torch.no_grad():
                m(x, ei, ew, h, c)
        finally:
            ops.LSTM_WIDE_ROWS_GEMM_NODES = saved
    return dict(eager=infer, graph=capture(infer), launches=launches(infer))


def chickenpox_epoch(name, fused):
    ei, ew, X, Y = chickenpox_train_split()
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV)
    m, opt = _model(name, 4, fused)

    def epoch():
        h = c = None
        cost = 0
        for t in range(X.size(0)):
            h, c = m.recurrent(X[t], ei, ew, h, c)
            cost = cost + torch.mean((m.linear(torch.relu(h)) - Y[t]) ** 2)
        (cost / X.size(0)).backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
    return dict(eager=epoch, launches=launches(epoch))


def main():
    g = load(os.path.join(ROOT, "tests", "golden"))
    wiki = (g["edge_index"].to(DEV), g["edge_weight"].to(DEV))
    graphs = {1068: wiki, **{n: _random_graph(n) for n in NO_GRAD_SIZES}}
    gpu, pl, clk = card()
    groups = []                                                        # (what, {path: config}); the paths of a group alternate
    for name in MODULES:
        groups.append(((name, "wikimaths_step"), {p: wikimaths_step(name, p == "rows", wiki) for p in ("rows", "autograd")}))
        groups.append(((name, "chickenpox_epoch"), {p: chickenpox_epoch(name, p == "rows") for p in ("rows", "autograd")}))
        for n, graph in graphs.items():
            for cin in (4, 16, 14):
                if cin == 14 and n not in (1068, 50000):
                    continue
                other = "op_for_op" if cin % 4 else "gemm_lstm"
                groups.append(((name, f"no_grad_cin{cin}_n{n}"), {p: no_grad_cell(name, cin, graph, p) for p in ("rows", other)}))
    for run in range(args.runs):
        for (name, what), cfgs in groups:
            for path, c in cfgs.items():
                steps = max(1, args.steps // 10) if what == "chickenpox_epoch" else args.steps
                for mode in ("eager", "graph"):
                    if mode not in c:
                        continue
                    c[mode]()
                    ms = timed(c[mode], steps)
                    print(json.dumps(dict(module=name, what=what, path=path, mode=mode, run=run, ms=round(ms, 4), launches=c["launches"],
                                          gpu=gpu, power_limit_w=pl, max_sm_clock_mhz=clk)), flush=True)


if __name__ == "__main__":
    main()
