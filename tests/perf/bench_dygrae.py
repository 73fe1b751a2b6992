"""DyGrEncoder on the device: the row-split GatedGraphConv + LSTM kernels (fused) against the op-for-op path (`fused_training = False` for
training; for inference the module's private op-for-op convolution followed by its torch.nn.LSTM), alternated, three runs each, eager and
CUDA-graph replay, on
* the tutorial epoch (dygrencoder_example.py: DyGrEncoder(4, 1, aggr, 32, 1), 103 chickenpox snapshots) with mean, add and max,
* a WikiMaths training step at (16, 2, "max", 64, 1) and (32, 1, "mean", 32, 1),
* no_grad steps of DyGrEncoder(16, 2, "mean", 32, 1) on 1 068 and 50 000 nodes.
Prints the card's name and power limit first.    python tests/perf/bench_dygrae.py"""
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from dygrae_seq import RecurrentDyGr, run  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import DyGrEncoder  # noqa: E402
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
    wei, wew, wX, wY = w["edge_index"].to(DEV), w["edge_weight"].to(DEV), w["X"].to(DEV), w["Y"].to(DEV)
    out = {}

    def epoch(aggr):
        m = RecurrentDyGr(DyGrEncoder, 4, 1, aggr, 32, 1).to(DEV)

        def make(fused):
            def step():
                m.recurrent.fused_training = fused
                m.zero_grad(set_to_none=False)
                _, cost = run(m, X, Y, ei, ew)
                cost.backward()
            return step
        return make
    for aggr in ("mean", "add", "max"):
        out[f"tutorial_epoch_{aggr}"] = (epoch(aggr), False)

    def wiki_step(C, Lg, aggr, Ho):
        m = RecurrentDyGr(DyGrEncoder, C, Lg, aggr, Ho, 1).to(DEV)

        def make(fused):
            def step():
                m.recurrent.fused_training = fused
                m.zero_grad(set_to_none=False)
                h, _, _ = m.recurrent(wX[0], wei, wew)
                torch.mean((m.linear(torch.relu(h)).squeeze() - wY[0]) ** 2).backward()
            return step
        return make
    out["wikimaths_train_16_2_max_64"] = (wiki_step(16, 2, "max", 64), False)
    out["wikimaths_train_32_1_mean_32"] = (wiki_step(32, 1, "mean", 32), False)

    def no_grad_step(n):
        g = torch.Generator(device="cpu").manual_seed(n)
        e = 8 * n
        cei = torch.randint(0, n, (2, e), generator=g).to(DEV)
        m = DyGrEncoder(16, 2, "mean", 32, 1).to(DEV)
        x = torch.randn(n, 14, generator=g).to(DEV)
        h = torch.randn(n, 32, generator=g).to(DEV)

        def make(fused):
            def step():
                with torch.no_grad():
                    if fused:
                        m(x, cei, None, h, h)
                    else:
                        plan = m._plan(cei, None, n)
                        m.recurrent_layer(m._conv_op_for_op(plan, x, cei, None)[None], (h[None], h[None]))
            return step
        return make
    out["no_grad_step_1068"] = (no_grad_step(1068), True)
    out["no_grad_step_50000"] = (no_grad_step(50000), True)
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
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
