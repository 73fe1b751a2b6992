"""TGCN training with the hidden state carried, the model of the reference's TGCN index-batching scripts (BatchedTGCN: TGCN2(2, 32, 1)
called once per step over a 12-step window, ReLU, Linear(32, 2); masked MAE, Adam; tgcn/metr_la_main.py).  One JSON line with the card,
its power limit (read in the same run) and, on the METR-LA (207 nodes) and PEMS-BAY (325 nodes) shapes at B = 64:
* ms per training step (forward, loss, backward, Adam) on the fused path (k_tgcn_attn + k_tgcn_attn_bwd / k_tgcn_cell_bwd) and on the
  op-for-op autograd path (`fused_training = False`), eager and replayed from a CUDA graph; the two paths alternate within the run,
  `--runs` times each;
* library launches per eager step of each path (libstmp kernels only: the autograd path's GEMMs and gate ops run in cuBLAS / torch);
* the largest loss and gradient differences between the two paths on the first step from the same weights (gradients also relative to
  the largest gradient of that tensor)."""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=30)
ap.add_argument("--runs", type=int, default=2)
args = ap.parse_args()
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

import torch  # noqa: E402

from pytorch_geometric_temporal_b200 import _lib, ops  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import TGCN2  # noqa: E402

DEV = "cuda"


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = None
    return torch.cuda.get_device_name(), (float(pl) if pl else None)


class BatchedTGCN(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.tgnn = TGCN2(2, 32, 1)
        self.linear = torch.nn.Linear(32, 2)

    def forward(self, x, edge_index, edge_weight):        # x (B, N, F, T) -> (B, T, N, 2)
        h, outs = None, []
        for t in range(x.shape[-1]):
            h = self.tgnn(x[..., t], edge_index, edge_weight, h)
            outs.append(self.linear(torch.relu(h)).unsqueeze(1))
        return torch.cat(outs, dim=1)


def timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def first_step(m, X, Y, ei, ew, mean, std):
    """Loss and gradients of the first step from the shared weights, detached: nothing of its autograd graph outlives the call (a
    graph kept alive would pin its AccumulateGrad nodes to the default stream and break the capture on the side stream)."""
    m.zero_grad()
    loss = ops.masked_mae(m(X, ei, ew) * std + mean, Y)
    loss.backward()
    return loss.detach(), [p.grad.detach().clone() for p in m.parameters()]


def shape(name, make):
    ei, ew, series = make(0, 1024)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    raw = torch.from_numpy(series).to(DEV)
    mean, std = raw.mean(dim=(0, 1)), raw.std(dim=(0, 1))
    starts = torch.randint(0, 1024 - 24, (64,), generator=torch.Generator().manual_seed(0)).to(DEV)
    s = (raw - mean) / std
    X = ops.window_gather(s, starts, 12, with_target=False).permute(0, 2, 3, 1).contiguous()     # (B, N, F, T), as the scripts permute
    Y = ops.window_gather(raw, starts + 12, 12, with_target=False)                               # (B, T, N, F)
    torch.manual_seed(0)
    init = BatchedTGCN().state_dict()
    paths = {}
    for path, fused in (("fused", True), ("autograd", False)):
        m = BatchedTGCN().to(DEV)
        m.load_state_dict(init)
        m.tgnn.fused_training = fused
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)

        def step(m=m, opt=opt):
            opt.zero_grad(set_to_none=False)
            loss = ops.masked_mae(m(X, ei, ew) * std + mean, Y)
            loss.backward()
            opt.step()
            return loss

        first = first_step(m, X, Y, ei, ew, mean, std)
        step()
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        step()
        torch.cuda.synchronize()
        paths[path] = dict(m=m, step=step, first=first, launches=_lib.launch_count() - n0)
    (lf, gf), (la, ga) = paths["fused"]["first"], paths["autograd"]["first"]
    res = {"loss_abs_diff": abs(float(lf - la)),
           "grad_max_abs_diff": max(float((a - b).abs().max()) for a, b in zip(gf, ga)),
           "grad_max_rel_diff": max(float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)) for a, b in zip(gf, ga))}
    for path, p in paths.items():
        res[f"{path}_launches_per_step"] = p["launches"]
        try:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(3):
                    p["step"]()
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                p["step"]()
            p["graph"] = g
        except RuntimeError as e:
            p["graph"] = None
            res[f"{path}_graph_ms"] = f"capture failed: {str(e).splitlines()[0][:120]}"
    for kind in ("eager", "graph"):
        for r in range(args.runs):
            for path, p in paths.items():             # alternate the two paths
                if kind == "eager":
                    ms = timed(p["step"], args.steps)
                elif p["graph"] is not None:
                    ms = timed(p["graph"].replay, args.steps)
                else:
                    continue
                res.setdefault(f"{path}_{kind}_ms", []).append(round(ms, 3))
    return {f"{name}_{k}": v for k, v in res.items()}


def main():
    gpu, plimit = card()
    out = {"bench": "tgcn_train", "model": "BatchedTGCN: TGCN2(2,32,1) + ReLU + Linear(32,2), T=12, masked MAE, Adam", "B": 64,
           "gpu": gpu, "power_limit_w": plimit}
    for name, make in (("metr_la", synthetic.metr_la_like), ("pems_bay", synthetic.pems_bay_like)):
        out.update(shape(name, make))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
