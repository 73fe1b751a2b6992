"""GMAN on the device: the fused attention kernels against the op-for-op route (every attention's core replaced by the reference's
algebra), alternated, three runs each, on
* the reference's unit-test shape: GMAN(1, 8, 8, 12, ...) on 50 nodes, B = 32, 12 history and 10 predicted steps,
* the PEMS-BAY shape (325 nodes, 12 + 12 steps, 8 heads of width 8) at B = 16 with L = 1 and L = 3,
* 1 024 nodes at B = 8, L = 1.
For each: a no_grad call (eager), a training step (forward, MAE, backward, Adam) eager and replayed from a CUDA graph, and the peak
memory of one eager training step.  Then a torch.profiler run of the fused PEMS-BAY L = 1 training step splits the CUDA time between
the attention kernels and everything else (the FC / BatchNorm layers, the gated fusion, Adam).
Prints the card's name and power limit first, then one JSON line per workload.    python tests/perf/bench_gman.py"""
import json
import os
import subprocess
import sys
import tempfile
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from pytorch_geometric_temporal_b200.nn.attention import GMAN  # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import gman as G  # noqa: E402

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


def _op_core(self, query, key, value, mask=False):
    if self.kind == "spatial":
        return G.spatial_attention_core(query, key, value, self._K, self._d)
    return G.temporal_attention_core(query, key, value, self._K, self._d, mask)


def _model(fused, L, N, B, his, pred):
    torch.manual_seed(0)
    m = GMAN(L, 8, 8, his, 0.1, 288, True, False).to(DEV)
    if not fused:
        for a in m.modules():
            if isinstance(a, G._Attention):
                a._core = types.MethodType(_op_core, a)
    X = torch.rand(B, his, N, device=DEV)
    SE = torch.randn(N, 64, device=DEV)
    TE = torch.stack((torch.randint(0, 7, (B, his + pred)), torch.randint(0, 288, (B, his + pred))), -1).float().to(DEV)
    Y = torch.rand(B, pred, N, device=DEV)
    return m, X, SE, TE, Y


def _graphed(fn):
    """fn captured in a CUDA graph after a warm-up on a side stream; the replay holds fn (the graph reads and writes its tensors)."""
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


def _step_fn(m, X, SE, TE, Y, capturable):
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=capturable)

    def step():
        opt.zero_grad(set_to_none=False)
        (m(X, SE, TE) - Y).abs().mean().backward()
        opt.step()
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    return step


def _call(fused, shape):
    m, X, SE, TE, _ = _model(fused, *shape)
    m.eval()

    def call():
        with torch.no_grad():
            m(X, SE, TE)
    return call


def _train(fused, shape, graph):
    m, X, SE, TE, Y = _model(fused, *shape)
    step = _step_fn(m, X, SE, TE, Y, capturable=graph)
    return _graphed(step) if graph else step


def _peak(fused, shape):
    step = _train(fused, shape, False)
    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


# (L, N, B, num_his, num_pred)
SHAPES = {
    "unit test shape: L = 1, N = 50, B = 32, 12 + 10 steps": ((1, 50, 32, 12, 10), 20),
    "PEMS-BAY: L = 1, N = 325, B = 16, 12 + 12 steps": ((1, 325, 16, 12, 12), 10),
    "PEMS-BAY: L = 3, N = 325, B = 16, 12 + 12 steps": ((3, 325, 16, 12, 12), 5),
    "N = 1024, L = 1, B = 8, 12 + 12 steps": ((1, 1024, 8, 12, 12), 5),
}


def _profile_split():
    """CUDA kernel time of one fused PEMS-BAY L = 1 training step, split into the attention kernels and the rest."""
    step = _train(True, SHAPES["PEMS-BAY: L = 1, N = 325, B = 16, 12 + 12 steps"][0], False)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            step()
        torch.cuda.synchronize()
    att = rest = 0.0
    for e in prof.key_averages():              # CUDA activity only: every entry is a kernel, copy or memset
        t = e.device_time_total
        if "k_gman_attn" in e.key:
            att += t
        else:
            rest += t
    out = os.path.join(os.environ.get("GMAN_BENCH_OUT", tempfile.gettempdir()), "gman_profile.txt")
    with open(out, "w") as f:
        f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40))
    return {"workload": "profile: fused PEMS-BAY L = 1 training step, CUDA time per step", "attention_kernels_ms": round(att / 5e3, 3),
            "other_kernels_ms": round(rest / 5e3, 3), "table": out}


def main():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(q.stdout.strip() or torch.cuda.get_device_name(0))
    for name, (shape, iters) in SHAPES.items():
        res = {}
        for what, make in (("no_grad_call_ms", lambda f: _call(f, shape)), ("train_step_eager_ms", lambda f: _train(f, shape, False)),
                           ("train_step_graph_ms", lambda f: _train(f, shape, True))):
            fns = {f: make(f) for f in (True, False)}
            r = {True: [], False: []}
            for _ in range(3):
                for f in (True, False):
                    r[f].append(round(_timed(fns[f], iters), 3))
            res[what] = {"fused": r[True], "op_for_op": r[False]}
            del fns
            torch.cuda.empty_cache()
        pk = {True: [], False: []}
        for _ in range(2):
            for f in (True, False):
                pk[f].append(_peak(f, shape))
                torch.cuda.empty_cache()
        res["train_step_peak_MiB"] = {"fused": pk[True], "op_for_op": pk[False]}
        print(json.dumps({"workload": name, **res}), flush=True)
    print(json.dumps(_profile_split()), flush=True)


if __name__ == "__main__":
    main()
