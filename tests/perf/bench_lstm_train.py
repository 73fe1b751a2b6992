"""The reference's LSTM tutorials on the row-split LSTM cell kernel (stmp_lstm_rows_*, DESIGN §4j) against today's op-for-op path:
* epoch      -- examples/recurrent/gconvlstm_example.py / gclstm_example.py: RecurrentGCN = GConvLSTM or GCLSTM(4, 32, K) + ReLU +
                Linear(32, 1) over the 103 snapshots of the 20 % chickenpox train split, H and C carried from None, cumulative MSE / 103,
                one backward and one Adam(lr = 0.01) step; K = 1 (the examples) and K = 2
* wiki_step  -- a WikiMaths-sized training step: (14, 32, 2) on the 1068-node WikiMaths graph (tests/golden/gconvgru_wikimaths.pt.gz) with
                seeded features, H = C = None, MSE, backward and one Adam step
* no_grad    -- one cell with H and C given at both sizes (chickenpox 20 nodes, cin 4; WikiMaths 1068 nodes, cin 14), K = 2
`fused` is the row-split kernel; `autograd` is the path the same module takes without it (op-for-op autograd for training; for inference
the basis assembly + wgmma `gemm_lstm` where (K(cin+32)) % 4 == 0, else op for op).  Each runs eagerly and replayed from a CUDA graph.
Configurations alternate within a run, `--runs` times each; every timed run prints one JSON line: ms per call, the card, its power limit
and maximum SM clock (read in the same run), and the library launches per eager call."""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=200, help="timed calls per run of the step and cell workloads")
ap.add_argument("--epochs", type=int, default=10, help="timed calls per run of the epoch workloads")
ap.add_argument("--runs", type=int, default=3)
args = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from pytorch_geometric_temporal_b200 import _lib  # noqa: E402
import lstm_seq  # noqa: E402

DEV = "cuda"
GOLDEN = os.path.join(ROOT, "tests", "golden")


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


def _model(module, F, K, fused):
    torch.manual_seed(1)
    m = lstm_seq.RecurrentGCN(lstm_seq.MODULES[module], F, K).to(DEV)
    if not fused:                        # every call, training or not, on the path the module takes without the row-split kernel
        m.recurrent._rows_ok = lambda *a, **k: False
    return m


def _entry(fn):
    return dict(eager=fn, graph=capture(fn), launches=launches(fn))


def epoch(module, K, fused, data):
    ei, ew, X, Y = data
    m = _model(module, 4, K, fused)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)

    def step():
        _, cost = lstm_seq.run(m, ei, ew, X, Y, device=DEV)
        cost.backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    return _entry(step)


def wiki_step(module, fused, graph):
    ei, ew = graph
    m = _model(module, 14, 2, fused)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    x = torch.randn(ei.max().item() + 1, 14, device=DEV)
    y = torch.randn(x.size(0), device=DEV)

    def step():
        h, _ = m.recurrent(x, ei, ew)
        cost = torch.mean((m.linear(torch.relu(h)).squeeze() - y) ** 2)
        cost.backward()
        opt.step()
        opt.zero_grad(set_to_none=False)
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    return _entry(step)


def cell(module, F, fused, graph):
    ei, ew = graph
    m = _model(module, F, 2, fused)
    N = ei.max().item() + 1
    x, h, c = torch.randn(N, F, device=DEV), torch.randn(N, 32, device=DEV) * 0.5, torch.randn(N, 32, device=DEV)

    def infer():
        with torch.no_grad():
            m.recurrent(x, ei, ew, h, c)
    return _entry(infer)


def main():
    gpu, plimit, clk = card()
    ei, ew, X, Y, _, _ = lstm_seq.data("chickenpox", GOLDEN)
    pox = (ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV))
    wei, wew, _, _, _, _ = lstm_seq.data("wikimaths", GOLDEN)
    wiki = (wei.to(DEV), wew.to(DEV))
    cfgs = {}
    for module in lstm_seq.MODULES:
        for fused in (True, False):
            path = "fused" if fused else "autograd"
            for K in (1, 2):
                cfgs[("chickenpox_epoch", f"{module}(4, 32, {K})", path)] = (epoch(module, K, fused, pox), args.epochs)
            cfgs[("wikimaths_train_step", f"{module}(14, 32, 2)", path)] = (wiki_step(module, fused, wiki), args.steps)
            cfgs[("no_grad_cell_chickenpox", f"{module}(4, 32, 2)", path)] = (cell(module, 4, fused, pox[:2]), args.steps)
            cfgs[("no_grad_cell_wikimaths", f"{module}(14, 32, 2)", path)] = (cell(module, 14, fused, wiki), args.steps)
    for r in range(args.runs):
        for mode in ("eager", "graph"):
            for (bench, model, path), (c, n) in cfgs.items():
                ms = timed(c[mode], n)
                print(json.dumps({"bench": bench, "model": model, "path": path, "mode": mode, "run": r, "ms_per_call": round(ms, 4),
                                  "library_launches_per_call": c["launches"], "gpu": gpu, "power_limit_w": plimit,
                                  "max_sm_clock_mhz": clk}), flush=True)


if __name__ == "__main__":
    main()
