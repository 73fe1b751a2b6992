"""BatchedDCRNN(2, 64, K) at K = 2 and 3 -- the DCRNN paper's 64 recurrent units -- on the 64-wide row-split kernels
(stmp_dcrnn_wide_rows_*) against the tiled path they replace.  One run, the paths alternated three times per measurement; prints the card
and its power limit (read in the same run) and one JSON line per (shape, K):
* shapes: METR-LA (207 nodes), PEMS-BAY (325 nodes) and synthetic banded graphs (synthetic.banded_graph plus a ring) of 2 000 and 11 160
  nodes at about 8 edges per node, B = 64 windows of T = 12 steps;
* infer_ms:  a no_grad call, 64-wide row-split against the tiled loop;
* train_ms: a training step (forward, masked MAE, backward, FlatAdam), eager and replayed as one CUDA graph, against
  `_fused_training = False` (autograd through the tiled path).  The largest shapes may not fit both captured steps at once: such a
  record says "out of memory".
    python tests/perf/bench_dcrnn_wide_rows.py [--steps N] [--shapes metr_la,pems_bay,n2000,n11160] [--K 2,3]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--shapes", default="metr_la,pems_bay,n2000,n11160")
ap.add_argument("--K", default="2,3")
args = ap.parse_args()

import torch  # noqa: E402

from pytorch_geometric_temporal_b200 import distributed as D  # noqa: E402
from pytorch_geometric_temporal_b200 import ops  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN  # noqa: E402

DEV = "cuda"
B, T = 64, 12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        pl, clk = float(q[0]), float(q[1])
    except (OSError, subprocess.SubprocessError, ValueError, IndexError):
        pl = clk = None
    return torch.cuda.get_device_name(), pl, clk


def timed(fn, steps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def graph_of(n, seed):
    """synthetic.banded_graph at 7 edges per node plus a ring (every in- and out-degree >= 1): about 8 edges per node"""
    ei, ew = synthetic.banded_graph(n, 7 * n, span=32, seed=seed)
    ring = torch.arange(n)
    ei = torch.cat([torch.from_numpy(ei), torch.stack([ring, (ring + 1) % n])], 1)
    ew = torch.cat([torch.from_numpy(ew), torch.full((n,), 0.5)])
    return ei.to(DEV), ew.to(DEV)


def shape(name):
    if name in ("pems_bay", "metr_la"):
        ei, ew, _ = (synthetic.pems_bay_like if name == "pems_bay" else synthetic.metr_la_like)(0, 16)
        n = 325 if name == "pems_bay" else 207
        return n, torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    n = int(name[1:])
    return (n,) + graph_of(n, n)


def alternate(fns, steps):
    """{key: [ms, ms, ms]}: each fn timed three times, the keys alternated"""
    res = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            res[k].append(round(timed(fn, steps), 3))
            torch.cuda.empty_cache()
    return res


K = 3


def model():
    torch.manual_seed(0)
    return BatchedDCRNN(2, 64, K).to(DEV)


def infer(n, ei, ew):
    m = model()
    X = torch.randn(B, T, n, 2, device=DEV)

    def run(fused):
        def f():
            m._wrows_ok = (lambda *a: False) if not fused else BatchedDCRNN._wrows_ok.__get__(m)
            with torch.no_grad():
                m(X, ei, ew)
        return f
    return alternate({"wrows": run(True), "tiled": run(False)}, args.steps)


def train(n, ei, ew):
    X = torch.randn(B, T, n, 2, device=DEV)
    Y = torch.randn(B, T, n, 64, device=DEV).abs()

    def setup(fused):
        m = model()
        m._fused_training = fused
        opt = D.FlatAdam(D.FlatGradSync(m.parameters()), lr=1e-3)

        def step():
            ops.masked_mae(m(X, ei, ew), Y).backward()
            opt.step()
        step()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                step()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        return step, g.replay

    (se_r, gr_r), (se_t, gr_t) = setup(True), setup(False)
    return alternate({"wrows_eager": se_r, "tiled_eager": se_t, "wrows_graph": gr_r, "tiled_graph": gr_t}, max(2, args.steps // 2))


def main():
    global K
    gpu, pl, clk = card()
    print(json.dumps({"bench": "dcrnn_wide_rows", "gpu": gpu, "power_limit_w": pl, "max_sm_clock_mhz": clk}), flush=True)
    for name in args.shapes.split(","):
        n, ei, ew = shape(name)
        for K in map(int, args.K.split(",")):
            rec = {"shape": name, "K": K, "nodes": n, "edges": int(ei.size(1)), "B": B, "T": T}
            rec["infer_ms"] = infer(n, ei, ew)
            try:
                rec["train_ms"] = train(n, ei, ew)
            except torch.cuda.OutOfMemoryError as e:             # both captured steps of the largest shape may not fit together
                rec["train_ms"] = f"out of memory: {str(e).splitlines()[0][:120]}"
            print(json.dumps(rec), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
