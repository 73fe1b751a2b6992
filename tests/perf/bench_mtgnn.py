"""MTGNN on the device: the fused graph kernels against the op-for-op route (fused_training = False for training, and the dense
reference algebra for the no_grad call), alternated, three runs each, on
* the reference test's shape: 207 nodes, B = 16, 12 steps, 3 layers, conv / residual channels 32, gcn_depth 2, k = 20,
* the METR-LA shape (207 nodes) and the PEMS-BAY shape (325 nodes) at B = 64, otherwise as above,
* the Traffic shape: 862 nodes, B = 16, 168 steps, 5 layers, dilation exponential 2, conv / residual channels 16, skip 32, end 64.
For each: a no_grad call and a training step (forward, MAE, backward, capturable Adam), both replayed from CUDA graphs, and the peak
memory of one training step.  Then torch.profiler runs of the fused training step at the METR-LA and Traffic shapes split the CUDA time between
the propagation kernels (k_mtgnn_*) and everything else.
Prints the card's name and power limit first, then one JSON line per workload.    python tests/perf/bench_mtgnn.py [--quick | --profile-only]"""
import json
import os
import re
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from pytorch_geometric_temporal_b200.nn.attention import MTGNN  # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import mtgnn as M  # noqa: E402

DEV = torch.device("cuda:0")
_BASE = dict(gcn_true=True, build_adj=True, gcn_depth=2, kernel_set=[2, 3, 6, 7], kernel_size=7, dropout=0.3, subgraph_size=20,
             node_dim=40, dilation_exponential=1, conv_channels=32, residual_channels=32, skip_channels=64, end_channels=128,
             seq_length=12, in_dim=2, out_dim=12, layers=3, propalpha=0.05, tanhalpha=3, layer_norm_affline=True)
WORKLOADS = {
    "reference_test": (dict(_BASE, num_nodes=207), 16),
    "metr_la": (dict(_BASE, num_nodes=207), 64),
    "pems_bay": (dict(_BASE, num_nodes=325), 64),
    "traffic": (dict(_BASE, num_nodes=862, seq_length=168, layers=5, dilation_exponential=2, conv_channels=16, residual_channels=16,
                     skip_channels=32, end_channels=64, in_dim=1, out_dim=1), 16),
}


def _graphed(fn, iters):
    """Mean ms per replay of fn captured as a CUDA graph (after warm-up on a side stream)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


class _OpForOp:
    """Routes every call of the model op for op (the reference's dense algebra on the GPU)."""

    def __init__(self, m):
        self.m = m

    def __enter__(self):
        self.orig = M.fused_route
        M.fused_route = lambda *a: False

    def __exit__(self, *exc):
        M.fused_route = self.orig


def _setup(cfg, B):
    torch.manual_seed(0)
    m = MTGNN(**cfg).to(DEV)
    X = torch.rand(B, cfg["in_dim"], cfg["num_nodes"], cfg["seq_length"], device=DEV)
    Y = torch.rand(B, cfg["out_dim"], cfg["num_nodes"], 1, device=DEV)
    opt = torch.optim.Adam(m.parameters(), lr=1e-4, capturable=True)
    return m, X, Y, opt


def _measure(cfg, B, fused, iters):
    m, X, Y, opt = _setup(cfg, B)

    def infer():
        with torch.no_grad():
            return m(X)

    def train():
        opt.zero_grad(set_to_none=False)
        (m(X) - Y).abs().mean().backward()
        opt.step()

    ctx = _OpForOp(m) if not fused else None
    if ctx:
        ctx.__enter__()
    try:
        m.eval()
        t_inf = _graphed(infer, iters)
        m.train()
        t_train = _graphed(train, iters)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        train()
        torch.cuda.synchronize()
        peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    finally:
        if ctx:
            ctx.__exit__(None, None, None)
    del m, X, Y, opt
    torch.cuda.empty_cache()
    return t_inf, t_train, peak


def _profile(cfg, B):
    m, X, Y, opt = _setup(cfg, B)

    def train():
        opt.zero_grad(set_to_none=False)
        (m(X) - Y).abs().mean().backward()
        opt.step()

    for _ in range(2):
        train()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            train()
        torch.cuda.synchronize()
    total, prop, top = 0.0, {}, []
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        total += t
        name = re.search(r"k_mtgnn_\w+", e.key)
        if name:
            prop[name.group(0)] = prop.get(name.group(0), 0.0) + t / 3e3
        else:
            top.append((t / 3e3, e.key[:60]))
    top.sort(reverse=True)
    return dict(total_ms=round(total / 3e3, 3), mtgnn_kernels_ms=round(sum(prop.values()), 3),
                per_kernel_ms={k: round(v, 3) for k, v in prop.items()}, top_other_ms=[(round(t, 3), k) for t, k in top[:6]])


def main():
    quick = "--quick" in sys.argv
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(card=q.stdout.strip())), flush=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    names = [] if "--profile-only" in sys.argv else ["reference_test", "traffic"] if quick else list(WORKLOADS)
    for name in names:
        cfg, B = WORKLOADS[name]
        iters = 5 if name == "traffic" else 20
        runs = {"fused": [], "op": []}
        for _ in range(3):
            for route in ("fused", "op"):
                runs[route].append(_measure(cfg, B, route == "fused", iters))
        res = dict(workload=name, B=B, N=cfg["num_nodes"])
        for route, rs in runs.items():
            res[route] = dict(no_grad_ms=[round(r[0], 3) for r in rs], train_ms=[round(r[1], 3) for r in rs],
                              train_peak_mib=round(rs[0][2], 1))
        print(json.dumps(res), flush=True)
    for name in ("metr_la", "traffic"):
        cfg, B = WORKLOADS[name]
        print(json.dumps(dict(profile=f"{name} fused training step", **_profile(cfg, B))), flush=True)


if __name__ == "__main__":
    main()
