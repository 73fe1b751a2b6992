"""MPNNLSTM on the device: the row-split kernels (fused) against the op-for-op route (the module's `_fused_ok` returning False), alternated,
three runs each, on
* the tutorial epoch as mpnnlstm_example.py writes it (MPNNLSTM(4, 32, 20, 1, 0.5), ReLU, Linear(68, 1), the 103 chickenpox training
  snapshots with autograd, cumulative MSE, one backward, an Adam step; eager),
* a WikiMaths training step (MPNNLSTM(14, 32, 1068, 1, 0.5), one call, one backward),
* the tutorial's 413 test snapshots in eval mode under no_grad (the example's eval pass runs with autograd enabled, which is the training
  route's forward; this workload is the no_grad one),
* 103 no_grad calls in training mode (dropout, BatchNorm batch statistics and running updates) on the tutorial's training snapshots,
* a no_grad call at window = 4, B = 16 on the 207-node METR-LA-like synthetic graph (13 248 rows), eval mode,
* a no_grad eval call on 50 000 nodes (in_channels 14), both routes under CUDA-graph replay.
Prints the card's name and power limit first, then one JSON line per workload.    python tests/perf/bench_mpnnlstm.py"""
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from mpnnlstm_seq import RecurrentMPNN, chickenpox  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import MPNNLSTM  # noqa: E402

DEV = torch.device("cuda:0")


def _timed(fn, iters):
    """Mean ms per call of fn over `iters` calls after one warm-up, by CUDA events."""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _route(m, fused):
    if not fused:
        m.fused_training = False
        m._fused_ok = lambda *a: False
    return m


def _tutorial(fused, training):
    ei, ew, train, test = chickenpox()
    X = (train if training else test)[0].to(DEV)
    ei, ew = ei.to(DEV), ew.to(DEV)
    torch.manual_seed(0)
    m = RecurrentMPNN(MPNNLSTM(4, 32, 20, 1, 0.5), 68).to(DEV).train(training)
    _route(m.recurrent, fused)

    def epoch():
        with torch.no_grad():
            for x in X:
                m(x, ei, ew)
    return epoch


def _train_epoch(fused):
    ei, ew, (X, Y), _ = chickenpox()
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV)
    torch.manual_seed(0)
    m = RecurrentMPNN(MPNNLSTM(4, 32, 20, 1, 0.5), 68).to(DEV).train()
    _route(m.recurrent, fused)
    opt = torch.optim.Adam(m.parameters(), lr=0.01)

    def epoch():
        cost = 0
        for t in range(X.shape[0]):
            cost = cost + torch.mean((m(X[t], ei, ew) - Y[t]) ** 2)
        (cost / X.shape[0]).backward()
        opt.step()
        opt.zero_grad()
    return epoch


def _wikimaths_step(fused):
    from wikimaths_seq import load as load_wikimaths
    w = load_wikimaths(os.path.join(os.path.dirname(HERE), "golden"))
    ei, ew, X, Y = w["edge_index"].to(DEV), w["edge_weight"].to(DEV), w["X"][0].to(DEV), w["Y"][0].to(DEV)
    torch.manual_seed(0)
    m = RecurrentMPNN(MPNNLSTM(14, 32, 1068, 1, 0.5), 78).to(DEV).train()
    _route(m.recurrent, fused)

    def step():
        torch.mean((m(X, ei, ew) - Y) ** 2).backward()
    return step


def _call(fused, rows_of, cin, nodes, window, graph_replay):
    ei, ew, rows = rows_of()
    torch.manual_seed(0)
    m = _route(MPNNLSTM(cin, 32, nodes, window, 0.5).to(DEV).eval(), fused)
    X = torch.randn(rows, cin, device=DEV)
    with torch.no_grad():
        if not graph_replay:
            return lambda: m(X, ei, ew)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(X, ei, ew)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = m(X, ei, ew)
    keep = (m, X, ei, ew, out)               # the graph reads the module's plan and these buffers: they must outlive it

    def replay():
        assert keep
        g.replay()
    return replay


def _metr(B=16, window=4):
    ei, ew, _ = synthetic.metr_la_like(0, 1)
    return torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV), B * window * 207


def _big(n=50000):
    g = torch.Generator().manual_seed(0)
    ei = torch.randint(0, n, (2, 8 * n), generator=g).to(DEV)
    return ei, torch.rand(8 * n, generator=g).to(DEV), n


WORKLOADS = {
    "tutorial epoch as written (103 training calls, backward, Adam; eager)": (_train_epoch, 3),
    "WikiMaths training step (1 068 nodes; eager)": (_wikimaths_step, 20),
    "413 eval calls under no_grad (tutorial test split, eager)": (lambda f: _tutorial(f, False), 3),
    "103 no_grad calls in training mode (eager)": (lambda f: _tutorial(f, True), 3),
    "window 4, B 16, METR-LA-like 207 nodes, no_grad eval call (eager)": (lambda f: _call(f, _metr, 2, 207, 4, False), 50),
    "50 000 nodes, no_grad eval call (CUDA-graph replay)": (lambda f: _call(f, _big, 14, 50000, 1, True), 50),
}


def main():
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(q.stdout.strip() or torch.cuda.get_device_name(0))
    for name, (make, iters) in WORKLOADS.items():
        res = {True: [], False: []}
        fns = {f: make(f) for f in (True, False)}
        for _ in range(3):
            for f in (True, False):
                res[f].append(round(_timed(fns[f], iters), 4))
        print(json.dumps({"workload": name, "fused_ms": res[True], "op_for_op_ms": res[False]}))


if __name__ == "__main__":
    main()
