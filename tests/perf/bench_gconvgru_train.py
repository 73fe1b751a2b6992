"""GConvGRU training epochs of the reference's tutorial (examples/recurrent/gconvgru_example.py, the project's config 1): RecurrentGCN =
GConvGRU(4, 32, K) + ReLU + Linear(32, 1) over the 20 % train split of the in-tree chickenpox data (103 snapshots of 20 nodes), the
cumulative MSE, one backward and one Adam(lr = 0.01) step per epoch.  For K in {1, 2} and two state patterns -- H = None at every
snapshot (the example) and H carried from snapshot to snapshot -- it times the fused path (stmp_gru_seq_fwd + stmp_gru_bwd_*) and the
op-for-op autograd path (`fused_training = False`), each eagerly and replayed from a CUDA graph.  The configurations alternate within the
run, `--runs` times each, and every timed run prints one JSON line: ms per epoch, the card and its power limit and maximum SM clock
(read in the same run), and the library launches of one eager epoch."""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--epochs", type=int, default=20, help="timed epochs per run")
ap.add_argument("--runs", type=int, default=3)
args = ap.parse_args()
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from pytorch_geometric_temporal_b200 import _lib  # noqa: E402
from gconvgru_seq import RecurrentGCN, chickenpox_train_split  # noqa: E402

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


def config(K, carried, fused, data):
    ei, ew, X, Y = data
    torch.manual_seed(K)
    m = RecurrentGCN(4, K).to(DEV)
    m.recurrent.fused_training = fused
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    H0 = torch.zeros(20, 32, device=DEV) if carried else None

    def epoch():
        opt.zero_grad(set_to_none=False)
        h, cost = H0, 0
        for t in range(X.shape[0]):
            hh = m.recurrent(X[t], ei, ew, h)
            if carried:
                h = hh
            cost = cost + torch.mean((m.linear(torch.relu(hh)) - Y[t]) ** 2)
        cost = cost / X.shape[0]
        cost.backward()
        opt.step()
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            epoch()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    epoch()
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        epoch()
    return dict(eager=epoch, graph=g.replay, launches=launches)


def main():
    gpu, plimit, clk = card()
    ei, ew, X, Y = chickenpox_train_split()
    data = (ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV))
    cfgs = {}
    for K in (1, 2):
        for carried in (False, True):
            for fused in (True, False):
                cfgs[(K, carried, fused)] = config(K, carried, fused, data)
    for c in cfgs.values():                  # warm every timed callable once more after all captures
        c["eager"]()
        c["graph"]()
    for r in range(args.runs):
        for mode in ("eager", "graph"):
            for (K, carried, fused), c in cfgs.items():      # alternate the configurations
                ms = timed(c[mode], args.epochs)
                print(json.dumps({"bench": "gconvgru_train", "K": K, "state": "carried" if carried else "none",
                                  "path": "fused" if fused else "autograd", "mode": mode, "run": r, "ms_per_epoch": round(ms, 3),
                                  "snapshots": int(X.shape[0]), "library_launches_per_eager_epoch": c["launches"], "gpu": gpu,
                                  "power_limit_w": plimit, "max_sm_clock_mhz": clk}), flush=True)


if __name__ == "__main__":
    main()
