#!/usr/bin/env python
"""The fused DCRNN forward alone at bench.py's headline shape: 1056 METR-LA-shaped windows (207 nodes, Cin 2, 12 steps) of
BatchedDCRNN(2, 32, K=2), one launch per call, timed with CUDA events over many launches.  Prints one JSON line: milliseconds per
launch (inference and with the training stash), the card and its power limit.  Run it with STMP_LIB pointed at another build to
compare two versions of the library."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from pytorch_geometric_temporal_b200 import _lib  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import BatchedDCRNN  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main(windows=1056, iters=100, reps=3):
    dev = torch.device("cuda", 0)
    ei, ew, _ = synthetic.metr_la_like(0, 16)
    ei, ew = torch.from_numpy(ei).to(dev), torch.from_numpy(ew).to(dev)
    torch.manual_seed(0)
    m = BatchedDCRNN(2, 32, 2).to(dev)
    X = torch.randn(windows, 12, 207, 2, device=dev)
    res = {"lib": _lib.LIB_PATH, "card": card(), "windows": windows}
    for name, grad in (("fwd_ms", False), ("fwd_stash_ms", True)):
        Xg = X.clone().requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            c0 = _lib.path_counters().get("k_dcrnn_seq_tc", 0)
            for _ in range(5):
                m(Xg, ei, ew)
            torch.cuda.synchronize()
            assert _lib.path_counters().get("k_dcrnn_seq_tc", 0) == c0 + 5, "the wgmma kernel did not serve the call"
            times = []
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    m(Xg, ei, ew)
                e1.record()
                torch.cuda.synchronize()
                times.append(round(e0.elapsed_time(e1) / iters, 4))
        res[name] = times
    print(json.dumps(res))


if __name__ == "__main__":
    main()
