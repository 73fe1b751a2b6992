"""AGCRN on the device: the fused kernels against the op-for-op route (the module's `_fused_ok` returning False), alternated, three runs
each, on
* the tutorial epoch as agcrn_example.py writes it (AGCRN(20, 8, 2, 2, 4), ReLU, Linear(2, 1), the 102 chickenpox training snapshots
  with h carried, cumulative MSE, one backward, an Adam step; eager),
* the paper's training step: AGCRN(307, 1, 64, 2, 10) and AGCRN(307, 64, 64, 2, 10) sharing a trained E over T = 12 steps of B = 64
  windows, Linear(64, 1), MSE, the backward and a capturable Adam step, replayed from a CUDA graph,
* a no_grad call of the second layer at that shape (B = 64, N = 307), replayed from a CUDA graph,
* a no_grad call of AGCRN(4096, 64, 64, 2, 10) at B = 4, replayed from a CUDA graph.
Prints the card's name and power limit first, then one JSON line per workload.    python tests/perf/bench_agcrn.py"""
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from agcrn_seq import chickenpox  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import AGCRN  # noqa: E402

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
        m._fused_ok = lambda *a: False
    return m


def _graphed(fn):
    """fn captured in a CUDA graph after a warm-up on a side stream; returns the replay.  The replay holds fn: the graph reads and
    writes the tensors fn closes over (model, inputs, optimizer state, gradients), so they must live as long as the graph."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()

    def replay():
        g.replay()
    replay.captured = fn
    return replay


def _tutorial(fused):
    X, Y = chickenpox()
    X, Y = X.view(-1, 1, 20, 8).to(DEV), Y.view(-1, 1, 20, 1).to(DEV)
    torch.manual_seed(0)
    rec, lin = _route(AGCRN(20, 8, 2, 2, 4), fused).to(DEV), torch.nn.Linear(2, 1).to(DEV)
    e = torch.empty(20, 4, device=DEV)
    torch.nn.init.xavier_uniform_(e)
    opt = torch.optim.Adam([*rec.parameters(), *lin.parameters()], lr=0.01)

    def epoch():
        h, cost = None, 0
        for t in range(X.shape[0]):
            h = rec(X[t], e, h)
            cost = cost + torch.mean((lin(torch.relu(h)) - Y[t]) ** 2)
        cost = cost / X.shape[0]
        cost.backward()
        opt.step()
        opt.zero_grad()
    return epoch


def _paper_step(fused):
    torch.manual_seed(0)
    layers = [_route(AGCRN(307, 1, 64, 2, 10), fused).to(DEV), _route(AGCRN(307, 64, 64, 2, 10), fused).to(DEV)]
    lin = torch.nn.Linear(64, 1).to(DEV)
    E = torch.nn.Parameter(torch.randn(307, 10, device=DEV))
    X, Y = torch.randn(64, 12, 307, 1, device=DEV), torch.randn(64, 307, 1, device=DEV)
    h0 = torch.zeros(64, 307, 64, device=DEV)
    params = [E, *layers[0].parameters(), *layers[1].parameters(), *lin.parameters()]
    opt = torch.optim.Adam(params, lr=1e-3, capturable=True)

    def step():
        opt.zero_grad(set_to_none=False)
        h1 = h2 = h0
        for t in range(12):
            h1 = layers[0](X[:, t], E, h1)
            h2 = layers[1](h1, E, h2)
        torch.mean((lin(h2) - Y) ** 2).backward()
        opt.step()
    for p in params:                         # gradients exist before capture, so the graph accumulates into fixed buffers
        p.grad = torch.zeros_like(p)
    return _graphed(step)


def _call(fused, N, B):
    torch.manual_seed(0)
    m = _route(AGCRN(N, 64, 64, 2, 10), fused).to(DEV)
    X, E, H = torch.randn(B, N, 64, device=DEV), torch.randn(N, 10, device=DEV), torch.randn(B, N, 64, device=DEV)

    def call():
        with torch.no_grad():
            m(X, E, H)
    return _graphed(call)


WORKLOADS = {
    "tutorial epoch as the example writes it (eager, backward and Adam step)": (_tutorial, 3),
    "paper training step, 2 layers x 12 steps, B = 64, N = 307 (CUDA-graph replay)": (_paper_step, 10),
    "no_grad call AGCRN(307, 64, 64, 2, 10), B = 64 (CUDA-graph replay)": (lambda f: _call(f, 307, 64), 50),
    "no_grad call AGCRN(4096, 64, 64, 2, 10), B = 4 (CUDA-graph replay)": (lambda f: _call(f, 4096, 4), 20),
}


def main():
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(q.stdout.strip() or torch.cuda.get_device_name(0))
    for name, (make, iters) in WORKLOADS.items():
        res = {True: [], False: []}
        fns = {f: make(f) for f in (True, False)}
        for _ in range(3):
            for f in (True, False):
                res[f].append(round(_timed(fns[f], iters), 4))
        print(json.dumps({"workload": name, "fused_ms": res[True], "op_for_op_ms": res[False]}), flush=True)
        del fns
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
