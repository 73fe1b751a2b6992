"""BatchedDCRNN on the row-split kernels against the paths they replace, at one width per run:
* 32:     BatchedDCRNN(2, 32, 2) on stmp_dcrnn_rows_*; shapes PEMS-BAY (325 nodes), random graphs of 2 000 and 11 160 nodes, METR-LA;
* narrow: BatchedDCRNN(2, 2, K), the reference's full-PeMS training model at K = 3, on stmp_dcrnn_narrow_rows_*; shapes banded graphs of
          2 000 and 11 160 nodes, PEMS-BAY;
* 64:     BatchedDCRNN(2, 64, K) at K = 2 and 3, the DCRNN paper's 64 recurrent units, on stmp_dcrnn_wide_rows_*; shapes METR-LA, PEMS-BAY,
          banded graphs of 2 000 and 11 160 nodes.
Synthetic graphs have about 8 edges per node (7 per node plus a ring, so every in- and out-degree is >= 1); B = 64 windows of T = 12
steps.  One run, the paths alternated three times per measurement; prints the card and its power limit (read in the same run) and one
JSON line per (shape, K):
* infer_ms:  a no_grad call, row-split against the tiled loop;
* train_ms: a training step (forward, masked MAE, backward, FlatAdam), eager and replayed as one CUDA graph, against
  `_fused_training = False` (autograd through the tiled path).  The largest shapes may not fit both captured steps at once: such a
  record says "out of memory";
* forward_ops_ms, on a shape the one-SM kernel (stmp_dcrnn_seq_fwd) serves -- where the module never takes the row-split route: the
  row-split forward called at ops level against that kernel.
    python tests/perf/bench_dcrnn_rows.py {32,narrow,64} [--steps N] [--shapes a,b,..] [--K 2,3]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
# width -> (bench name, arm name, out_channels, K list, shapes, synthetic graph family)
WIDTHS = {"32": ("dcrnn_rows", "rows", 32, "2", "pems_bay,n2000,n11160,metr_la", "random"),
          "narrow": ("dcrnn_narrow_rows", "nrows", 2, "3", "n2000,n11160,pems_bay", "banded"),
          "64": ("dcrnn_wide_rows", "wrows", 64, "2,3", "metr_la,pems_bay,n2000,n11160", "banded")}
ap = argparse.ArgumentParser()
ap.add_argument("width", choices=sorted(WIDTHS))
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--shapes", default=None)
ap.add_argument("--K", default=None, help="narrow: 1..4, 64: 2 and 3, 32: 2 only")
args = ap.parse_args()
if args.width == "32" and args.K not in (None, "2"):
    ap.error("the 32-wide row-split kernels serve K = 2 only")
BENCH, ARM, COUT, K_LIST, SHAPES, GRAPHS = WIDTHS[args.width]

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
    """7 edges per node -- uniformly random, or synthetic.banded_graph -- plus a ring"""
    ring = torch.arange(n)
    if GRAPHS == "random":
        g = torch.Generator().manual_seed(seed)
        ei = torch.cat([torch.randint(0, n, (2, 7 * n), generator=g), torch.stack([ring, (ring + 1) % n])], 1)
        ei = torch.unique(ei, dim=1)
        ei = ei[:, ei[0] != ei[1]]
        return ei.to(DEV), (torch.rand(ei.size(1), generator=g) + 0.1).to(DEV)
    ei, ew = synthetic.banded_graph(n, 7 * n, span=32, seed=seed)
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


def model(K):
    torch.manual_seed(0)
    return BatchedDCRNN(2, COUT, K).to(DEV)


def infer(K, n, ei, ew):
    m = model(K)
    X = torch.randn(B, T, n, 2, device=DEV)

    def run(fused):
        def f():
            m._rows_ok = (lambda *a: False) if not fused else BatchedDCRNN._rows_ok.__get__(m)
            with torch.no_grad():
                m(X, ei, ew)
        return f
    return alternate({ARM: run(True), "tiled": run(False)}, args.steps)


def train(K, n, ei, ew):
    X = torch.randn(B, T, n, 2, device=DEV)
    Y = torch.randn(B, T, n, COUT, device=DEV).abs()

    def setup(fused):
        m = model(K)
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
    return alternate({ARM + "_eager": se_r, "tiled_eager": se_t, ARM + "_graph": gr_r, "tiled_graph": gr_t}, max(2, args.steps // 2))


def forward_ops(K, n, ei, ew):
    m = model(K)
    X = torch.randn(B, T, n, 2, device=DEV)
    plan = m._plan(ei, ew, n)
    whsT, wzrT = m._rows_packed()
    p = m._params()
    wimg = m._weight_image()
    if COUT == 32:
        rows = lambda: ops.dcrnn_rows_fwd(plan, X, wzrT, whsT, *p[3:])            # noqa: E731
    else:
        rows = lambda: ops.dcrnn_hoisted_rows_fwd(plan, X, wzrT, whsT, *p[3:], K)  # noqa: E731
    with torch.no_grad():
        return alternate({ARM: rows, "one_sm": lambda: ops.dcrnn_seq_fwd(plan, X, *p, K, wimage=wimg)}, max(args.steps, 20))


def main():
    gpu, pl, clk = card()
    print(json.dumps({"bench": BENCH, "gpu": gpu, "power_limit_w": pl, "max_sm_clock_mhz": clk}), flush=True)
    for name in (args.shapes or SHAPES).split(","):
        n, ei, ew = shape(name)
        for K in map(int, (args.K or K_LIST).split(",")):
            rec = {"shape": name, "K": K, "nodes": n, "edges": int(ei.size(1)), "B": B, "T": T}
            if ops.dcrnn_seq_supported(model(K)._plan(ei, ew, n), 2, COUT, K):
                rec["forward_ops_ms"] = forward_ops(K, n, ei, ew)
            else:
                rec["infer_ms"] = infer(K, n, ei, ew)
                try:
                    rec["train_ms"] = train(K, n, ei, ew)
                except torch.cuda.OutOfMemoryError as e:             # both captured steps of the largest shape may not fit together
                    rec["train_ms"] = f"out of memory: {str(e).splitlines()[0][:120]}"
            print(json.dumps(rec), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
