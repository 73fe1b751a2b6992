"""EvolveGCNO / EvolveGCNH on the device: the row-split kernels (fused) against the op-for-op path (`fused_training = False` for training;
for inference a module with C > 32's route forced by `_fused_ok` returning False), alternated, three runs each, on
* both tutorial epochs as written (evolvegcno_example.py / evolvegcnh_example.py: 103 chickenpox snapshots, C = 4, eager),
* a WikiMaths training step at C = 14 (1 068 nodes, one call, one backward),
* a no_grad call on 50 000 nodes at C = 32, the fused route under CUDA-graph replay, op for op eagerly.
Prints the card's name and power limit first, then one JSON line per workload.    python tests/perf/bench_evolvegcn.py"""
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from evolvegcn_seq import RecurrentEGCN, run  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import EvolveGCNH, EvolveGCNO  # noqa: E402
from wikimaths_seq import load as load_wikimaths  # noqa: E402

DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(HERE), "golden")


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
    m.fused_training = fused
    if not fused:
        m._fused_ok = lambda *a: False          # inference too: the op-for-op route
    return m


def _tutorial(kind, fused):
    ei, ew, X, Y = chickenpox_train_split()
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV)
    torch.manual_seed(0)
    m = RecurrentEGCN(EvolveGCNH(20, 4) if kind == "H" else EvolveGCNO(4), 4).to(DEV)
    _route(m.recurrent, fused)
    opt = torch.optim.Adam(m.parameters(), lr=0.01)

    def epoch():
        run(m, X, Y, ei, ew, 1, retain=kind == "O")
        opt.step()
        opt.zero_grad()
    return epoch


def _wikimaths(kind, fused):
    w = load_wikimaths(GOLDEN)
    ei, ew, X = w["edge_index"].to(DEV), w["edge_weight"].to(DEV), w["X"][0].to(DEV)
    torch.manual_seed(0)
    m = _route((EvolveGCNH(1068, 14) if kind == "H" else EvolveGCNO(14)).to(DEV), fused)

    def step():
        m.weight = None
        m(X, ei, ew).square().mean().backward()
    return step


def _graph_call(kind, fused):
    n = 50000
    g = torch.Generator().manual_seed(1)
    ei = torch.randint(0, n, (2, 8 * n), generator=g).to(DEV)
    ew = torch.rand(8 * n, generator=g).to(DEV)
    X = torch.randn(n, 32, generator=g).to(DEV)
    torch.manual_seed(0)
    m = _route((EvolveGCNH(n, 32) if kind == "H" else EvolveGCNO(32)).to(DEV), fused)
    if not fused:
        def call():
            with torch.no_grad():
                m.weight = None
                m(X, ei, ew)
        return call
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                m.weight = None
                m(X, ei, ew)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        m.weight = None
        with torch.cuda.graph(graph):
            m(X, ei, ew)

    def replay():
        graph.replay()
    replay.operands = (m, X, ei, ew)           # the captured call reads them and the module's cached plan: they live as long as the graph
    return replay


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(f"# {card.strip()}")
    work = [("tutorial epoch", _tutorial, 3), ("WikiMaths training step C=14", _wikimaths, 50), ("no_grad call, 50 000 nodes, C=32, graph", _graph_call, 200)]
    for name, make, iters in work:
        for kind in ("O", "H"):
            fns = {fused: make(kind, fused) for fused in (True, False)}
            times = {True: [], False: []}
            for _ in range(3):
                for fused in (True, False):
                    times[fused].append(_timed(fns[fused], iters))
            print(json.dumps({"workload": name, "model": "EvolveGCN" + kind, "fused_ms": [round(t, 4) for t in times[True]],
                              "op_for_op_ms": [round(t, 4) for t in times[False]]}))


if __name__ == "__main__":
    main()
