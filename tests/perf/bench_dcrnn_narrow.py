"""Narrow-state DCRNN, the reference's index-batching training model BatchedDCRNN(2, 2, K=3): one JSON line with the card, its power
limit (read in the same run) and
* training: ms per step of the reference example's step at the PEMS-BAY shape (examples/indexBatching/DCRNN/pems_ddp.py): B = 64,
  T = 12, forward, masked MAE on de-normalised outputs, backward, Adam -- eager and replayed as one CUDA graph;
* inference: windows/s through forward_indexed at B = 64 and B = 1056 on the METR-LA and PEMS-BAY shapes.

To compare two builds, check each out, build it, and run this script once per checkout, alternating:
    python tests/perf/bench_dcrnn_narrow.py --repo <checkout> --dump <file.pt>
(--repo puts that checkout's package first on sys.path, so its own library and routing run.)  --dump saves the outputs and gradients
of the timed sizes for an fp32-tolerance comparison of the builds."""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--repo", default=os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--dump", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.repo))

import torch  # noqa: E402

from pytorch_geometric_temporal_b200 import ops  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN  # noqa: E402

DEV = "cuda"


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = None
    return torch.cuda.get_device_name(), (float(pl) if pl else None)


def timed(fn, steps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def training(dump):
    ei, ew, series = synthetic.pems_bay_like(0, 512)
    ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
    raw = torch.from_numpy(series).to(DEV)
    mean, std = raw.mean(dim=(0, 1)), raw.std(dim=(0, 1))
    s = (raw - mean) / std
    starts = torch.randint(0, 512 - 24, (64,), generator=torch.Generator().manual_seed(0)).to(DEV)
    X = ops.window_gather(s, starts, 12, with_target=False)
    Y = ops.window_gather(raw, starts + 12, 12, with_target=False)
    torch.manual_seed(0)
    m = BatchedDCRNN(2, 2, 3).to(DEV)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)

    first = {}

    def step():
        opt.zero_grad(set_to_none=False)
        out = m(X, ei, ew)
        loss = ops.masked_mae(out * std + mean, Y)
        loss.backward()
        if not first:                                           # outputs and gradients of the first step, for the comparison
            first.update(out=out.detach().cpu(), loss=loss.detach().cpu(), grads=[p.grad.cpu() for p in m.parameters()])
        opt.step()

    step()
    if dump is not None:
        dump["train_out"], dump["train_loss"], dump["train_grads"] = first["out"], first["loss"], first["grads"]
    eager = timed(step, args.steps)
    graph_ms = None
    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                step()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        graph_ms = timed(g.replay, args.steps) * 1e3
    except RuntimeError as e:                                   # a build whose training step cannot be captured
        graph_ms = f"capture failed: {str(e).splitlines()[0][:120]}"
    return eager * 1e3, graph_ms


def inference(dump):
    res = {}
    for name, make in (("metr_la", synthetic.metr_la_like), ("pems_bay", synthetic.pems_bay_like)):
        ei, ew, series = make(0, 2048)
        ei, ew = torch.from_numpy(ei).to(DEV), torch.from_numpy(ew).to(DEV)
        s = torch.from_numpy(series).to(DEV)
        torch.manual_seed(1)
        m = BatchedDCRNN(2, 2, 3).to(DEV)
        for B in (64, 1056):
            starts = torch.randint(0, 2048 - 12, (B,), generator=torch.Generator().manual_seed(B)).to(DEV)
            with torch.no_grad():
                out = m.forward_indexed(s, starts, 12, ei, ew)
                if dump is not None:
                    dump[f"infer_{name}_{B}"] = out.cpu()
                sec = timed(lambda: m.forward_indexed(s, starts, 12, ei, ew), max(args.steps, 20))
            res[f"{name}_B{B}_windows_per_s"] = round(B / sec, 1)
    return res


def main():
    name, plimit = card()
    dump = {} if args.dump else None
    eager_ms, graph_ms = training(dump)
    inf = inference(dump)
    if args.dump:
        torch.save(dump, args.dump)
    print(json.dumps({"bench": "dcrnn_narrow", "model": "BatchedDCRNN(2,2,K=3)", "repo": os.path.abspath(args.repo), "gpu": name,
                      "power_limit_w": plimit, "train_B64_T12_pems_bay_eager_ms": round(eager_ms, 3),
                      "train_B64_T12_pems_bay_graph_ms": round(graph_ms, 3) if isinstance(graph_ms, float) else graph_ms, **inf}))


if __name__ == "__main__":
    main()
