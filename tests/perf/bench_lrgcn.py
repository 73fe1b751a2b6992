"""LRGCN on the device: the row-split cell (fused) against the op-for-op path (`fused_training = False` for training; for inference the
op-for-op path is forced by a 3-D X of one batch), alternated, three runs each, eager and CUDA-graph replay, on
* the tutorial epoch (lrgcn_example.py: LRGCN(4, 32, 1, 1), 103 chickenpox snapshots, float edge_attr as edge_type) and the same with R = 2,
* a WikiMaths training step at (14, 32, 2, 2) and (14, 64, 1, 1),
* no_grad cells on 1 068 and 50 000 nodes.
Prints the card's name and power limit first.    python tests/perf/bench_lrgcn.py"""
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from lrgcn_seq import RecurrentLRGCN, run  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import LRGCN  # noqa: E402
from wikimaths_seq import load as load_wikimaths  # noqa: E402

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
    return a.elapsed_time(b) / iters * 1e3          # us


def _graphed(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def workloads():
    torch.manual_seed(0)
    ei, ew, X, Y = chickenpox_train_split()
    ei, ew, X, Y = ei.to(DEV), ew.to(DEV), X.to(DEV), Y.to(DEV)
    w = load_wikimaths(os.path.join(os.path.dirname(HERE), "golden"))
    wei, wX, wY = w["edge_index"].to(DEV), w["X"].to(DEV), w["Y"].to(DEV)
    wet = (wei[0] < wei[1]).long()
    out = {}

    def epoch(R, et):
        m = RecurrentLRGCN(LRGCN, 4, 32, R, 1).to(DEV)

        def make(fused):
            def step():
                m.recurrent.fused_training = fused
                m.zero_grad(set_to_none=False)
                _, cost = run(m, X, Y, ei, et)
                cost.backward()
            return step
        return make
    out["tutorial_epoch_R1"] = (epoch(1, ew), False)
    out["tutorial_epoch_R2"] = (epoch(2, (ei[0] < ei[1]).long()), False)

    def wiki_step(co, R, B, et):
        m = RecurrentLRGCN(LRGCN, 14, co, R, B).to(DEV)

        def make(fused):
            def step():
                m.recurrent.fused_training = fused
                m.zero_grad(set_to_none=False)
                h, c = m.recurrent(wX[0], wei, et)
                torch.mean((m.linear(torch.relu(h)).squeeze() - wY[0]) ** 2).backward()
            return step
        return make
    out["wikimaths_train_32_R2_B2"] = (wiki_step(32, 2, 2, wet), False)
    out["wikimaths_train_64_R1_B1"] = (wiki_step(64, 1, 1, torch.zeros_like(wet)), False)

    def cell(n):
        g = torch.Generator(device="cpu").manual_seed(n)
        e = 8 * n
        cei = torch.randint(0, n, (2, e), generator=g).to(DEV)
        cet = torch.randint(0, 2, (e,), generator=g).to(DEV)
        m = LRGCN(14, 32, 2, 2).to(DEV)
        x = torch.randn(n, 14, generator=g).to(DEV)
        h = torch.randn(n, 32, generator=g).to(DEV)

        def make(fused):
            xx = x if fused else x.unsqueeze(0)          # a batched X takes the op-for-op path
            hh = h if fused else h.unsqueeze(0)

            def step():
                with torch.no_grad():
                    m(xx, cei, cet, hh, hh)
            return step
        return make
    out["no_grad_cell_1068"] = (cell(1068), True)
    out["no_grad_cell_50000"] = (cell(50000), True)
    return out


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(json.dumps({"gpu": smi.strip(), "torch": torch.__version__}))
    for name, (make, graphable) in workloads().items():
        res = {"workload": name}
        iters = 3 if name.startswith("tutorial") else 20
        for mode in ("eager", "graph"):
            if mode == "graph" and not graphable:
                continue
            times = {True: [], False: []}
            for _ in range(3):
                for fused in (True, False):
                    fn = make(fused)
                    times[fused].append(_timed(_graphed(fn) if mode == "graph" else fn, iters))
            res[mode] = {"fused_us": sorted(times[True]), "op_for_op_us": sorted(times[False])}
        print(json.dumps(res))


if __name__ == "__main__":
    main()
