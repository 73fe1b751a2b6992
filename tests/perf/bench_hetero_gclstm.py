"""HeteroGCLSTM on the device: the fused one-launch inference kernel against the op-for-op route (the module's `_fused_ok` returning
False), alternated, three runs each, on
* the reference's unit-test shape (50 authors with 20 features, 50 papers with 30, out 32, writes + rev_writes): a no_grad call with H
  and C carried, eager;
* a seeded synthetic three-type graph where rows split across SMs: 200 000 users (16 features), 50 000 items (8), 2 000 shops (4),
  2 M edges over five edge types including a self-relation, out 32: a no_grad call with H and C carried, replayed from a CUDA graph;
* the unit-test shape's training step (backward and Adam), eager;
* a 12-snapshot training step on the synthetic graph (H / C carried, backward, capturable Adam), replayed from a CUDA graph.
Prints the card's name and power limit first, then one JSON line per workload.    python tests/perf/bench_hetero_gclstm.py"""
import json
import subprocess
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from pytorch_geometric_temporal_b200.nn.hetero import HeteroGCLSTM  # noqa: E402

DEV = torch.device("cuda:0")


def _timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _graphed(fn):
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
    replay.captured = fn            # the graph reads the tensors fn closes over: keep them alive
    return replay


def _model(types, edges, out, seed, fused):
    g = torch.Generator().manual_seed(seed)
    x = {t: torch.rand(n, c, generator=g).to(DEV) for t, (n, c) in types.items()}
    ei = {}
    for s, r, d, E in edges:
        ei[(s, r, d)] = torch.stack([torch.randint(0, types[s][0], (E,), generator=g), torch.randint(0, types[d][0], (E,), generator=g)]).to(DEV)
    m = HeteroGCLSTM({t: c for t, (_, c) in types.items()}, out, (list(types), list(ei))).to(DEV)
    if not fused:
        m._fused_ok = lambda *a: False
    h = {t: torch.rand(n, out, generator=g).to(DEV) for t, (n, _) in types.items()}
    c = {t: torch.rand(n, out, generator=g).to(DEV) for t, (n, _) in types.items()}
    return m, x, ei, h, c


UNIT = ({"author": (50, 20), "paper": (50, 30)}, [("author", "writes", "paper", 125), ("paper", "rev_writes", "author", 125)])
LARGE = ({"user": (200_000, 16), "item": (50_000, 8), "shop": (2_000, 4)},
         [("item", "bought_by", "user", 800_000), ("user", "follows", "user", 400_000), ("user", "buys", "item", 600_000),
          ("shop", "sells", "item", 100_000), ("item", "sold_by", "shop", 100_000)])


def _nograd(spec, fused, graphed, iters):
    m, x, ei, h, c = _model(*spec, 32, 0, fused)
    with torch.no_grad():
        m(x, ei, h, c)                                               # plans and packs
        fn = (lambda: m(x, ei, h, c))
        if graphed:
            fn = _graphed(fn)
        return _timed(fn, iters)


def _train(spec, fused, steps, graphed, iters):
    m, x, ei, h, c = _model(*spec, 32, 0, True)
    m.fused_training = fused
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=graphed)
    with torch.no_grad():
        m(x, ei, h, c)                                               # plans and packs

    def step():
        opt.zero_grad(set_to_none=False)
        hn, cn, loss = h, c, 0
        for _ in range(steps):
            hn, cn = m(x, ei, hn, cn)
            loss = loss + sum(v.square().mean() for v in hn.values())
        loss.backward()
        opt.step()
    return _timed(_graphed(step) if graphed else step, iters)


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": q.stdout.strip()}))
    work = [("unit no_grad call, eager", lambda f: _nograd(UNIT, f, False, 200)),
            ("synthetic 252k nodes / 2M edges no_grad call, CUDA graph", lambda f: _nograd(LARGE, f, True, 50)),
            ("unit training step, eager", lambda f: _train(UNIT, f, 1, False, 50)),
            ("synthetic 12-snapshot training step, CUDA graph", lambda f: _train(LARGE, f, 12, True, 5))]
    for name, fn in work:
        res = {"fused": [], "op_for_op": []}
        for _ in range(3):
            res["fused"].append(round(fn(True), 4))
            res["op_for_op"].append(round(fn(False), 4))
        print(json.dumps({"workload": name, "ms": res}))


if __name__ == "__main__":
    main()
