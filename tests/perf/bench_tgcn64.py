"""TGCN / A3TGCN training and inference at 64 hidden channels, fused (k_tgcn_wide_attn + k_tgcn_attn_bwd<NQ, 2> /
k_tgcn_wide_cell_bwd) against op-for-op (SpMM + cuBLAS + pointwise ops).  One JSON line with the card, its power limit (read in the same
run) and, on the METR-LA (207 nodes) and PEMS-BAY (325 nodes) shapes at B = 64, T = 12:
* BatchedTGCN, the model of the reference's TGCN index-batching scripts at hidden_dim 64 (TGCN2(2, 64, 1) called once per step with the
  state carried, ReLU, Linear(64, 2), masked MAE, Adam): ms per training step, eager and replayed from a CUDA graph, fused against
  `fused_training = False`, the two paths alternating `--runs` times each;
* the A3TGCN2 example's model at 64 channels (A3TGCN2(2, 64, 12) with H = None, ReLU, Linear(64, 12), masked MAE, Adam): the same;
* a `no_grad` forward of each model, fused against op-for-op (the module's 64-wide routes switched off for that call);
* library launches per eager training step of each path, and the largest loss and gradient differences between the two paths on the
  first step from the same weights."""
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
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN2, TGCN2  # noqa: E402

DEV = "cuda"
W = 64


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
        self.tgnn = TGCN2(2, W, 1)
        self.linear = torch.nn.Linear(W, 2)

    @property
    def base(self):
        return self.tgnn

    def forward(self, x, edge_index, edge_weight):        # x (B, N, F, T) -> (B, T, N, 2)
        h, outs = None, []
        for t in range(x.shape[-1]):
            h = self.tgnn(x[..., t], edge_index, edge_weight, h)
            outs.append(self.linear(torch.relu(h)).unsqueeze(1))
        return torch.cat(outs, dim=1)


class A3(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.tgnn = A3TGCN2(2, W, 12, 64)
        self.linear = torch.nn.Linear(W, 12)

    @property
    def base(self):
        return self.tgnn._base_tgcn

    def forward(self, x, edge_index, edge_weight):        # x (B, N, F, T) -> (B, T, N, 1)
        return self.linear(torch.relu(self.tgnn(x, edge_index, edge_weight))).permute(0, 2, 1).unsqueeze(-1)


def timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def workload(name, make, cls):
    ei, ew, series = make(0, 1024)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    raw = torch.from_numpy(series).to(DEV)
    mean, std = raw.mean(dim=(0, 1)), raw.std(dim=(0, 1))
    starts = torch.randint(0, 1024 - 24, (64,), generator=torch.Generator().manual_seed(0)).to(DEV)
    X = ops.window_gather((raw - mean) / std, starts, 12, with_target=False).permute(0, 2, 3, 1).contiguous()   # (B, N, F, T)
    Y = ops.window_gather(raw, starts + 12, 12, with_target=False)                                             # (B, T, N, F)
    if cls is A3:
        Y = Y[..., :1]
        mean, std = mean[:1], std[:1]
    torch.manual_seed(0)
    init = cls().state_dict()
    paths = {}
    for path, fused in (("fused", True), ("opforop", False)):
        m = cls().to(DEV)
        m.load_state_dict(init)
        m.base.fused_training = fused
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)

        def step(m=m, opt=opt):
            opt.zero_grad(set_to_none=False)
            loss = ops.masked_mae(m(X, ei, ew) * std + mean, Y)
            loss.backward()
            opt.step()
            return loss

        def infer(m=m, fused=fused):
            with torch.no_grad():
                if not fused:                         # the 64-wide routes off for this call: the op-for-op path
                    m.base._ATTN_WIDTHS = (32,)
                out = m(X, ei, ew)
                m.base.__dict__.pop("_ATTN_WIDTHS", None)
            return out

        out0 = infer()
        m.zero_grad()
        loss = ops.masked_mae(m(X, ei, ew) * std + mean, Y)
        loss.backward()
        first = (loss.detach(), [p.grad.detach().clone() for p in m.parameters()])
        del loss
        step()
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        step()
        torch.cuda.synchronize()
        paths[path] = dict(m=m, step=step, infer=infer, out0=out0, first=first, launches=_lib.launch_count() - n0)
    (lf, gf), (la, ga) = paths["fused"]["first"], paths["opforop"]["first"]
    res = {"loss_abs_diff": abs(float(lf - la)),
           "grad_max_abs_diff": max(float((a - b).abs().max()) for a, b in zip(gf, ga)),
           "grad_max_rel_diff": max(float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)) for a, b in zip(gf, ga)),
           "no_grad_max_abs_diff": float((paths["fused"]["out0"] - paths["opforop"]["out0"]).abs().max())}
    for path, p in paths.items():
        res[f"{path}_launches_per_step"] = p["launches"]
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
    for kind in ("eager", "graph", "no_grad"):
        for r in range(args.runs):
            for path, p in paths.items():             # alternate the two paths
                fn = p["step"] if kind == "eager" else (p["graph"].replay if kind == "graph" else p["infer"])
                res.setdefault(f"{path}_{kind}_ms", []).append(round(timed(fn, args.steps), 3))
    return {f"{name}_{k}": v for k, v in res.items()}


def main():
    gpu, plimit = card()
    out = {"bench": "tgcn64", "models": {"tgcn": "BatchedTGCN: TGCN2(2,64,1) + ReLU + Linear(64,2), T=12",
                                         "a3tgcn": "A3TGCN2(2,64,12) + ReLU + Linear(64,12)", "loss": "masked MAE", "optimizer": "Adam"},
           "B": 64, "gpu": gpu, "power_limit_w": plimit}
    for model, cls in (("tgcn", BatchedTGCN), ("a3tgcn", A3)):
        for name, make in (("metr_la", synthetic.metr_la_like), ("pems_bay", synthetic.pems_bay_like)):
            out.update(workload(f"{model}_{name}", make, cls))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
