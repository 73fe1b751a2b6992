#!/usr/bin/env python
"""Weight-gradient contraction of the DCRNN training step at the reference's batch size (rows = 12 * 64 * 207): fp32 FFMA kernel vs the
wgmma TF32-split kernel, both against a float64 contraction.  One JSON line."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from pytorch_geometric_temporal_b200 import _lib, ops  # noqa: E402

dev = torch.device("cuda", 0)
cin, Co, K = 2, 32, 2
rows = 12 * 64 * 207
C = cin + Co
ld = ops.dcrnn_bwd_basis_ld(cin, Co, K)
torch.manual_seed(0)
S1 = torch.randn(rows, 1, ld, device=dev)
S2 = torch.randn(rows, 1, ld, device=dev)
dpzr = torch.randn(rows, 2 * Co, device=dev) * 1e-4
dph = torch.randn(rows, Co, device=dev) * 1e-4
ref_zr = S1[:, 0, :3 * C].double().t() @ dpzr.double()
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
res = {}
for tc in (0, 1):
    _lib.set_option("dcrnn_wgrad_tc", tc)
    out = ops.dcrnn_bwd_wgrad(cin, K, S1, S2, dpzr, dph, True)
    got = torch.cat([out[0][0, 0], out[0][0, 1], out[0][1, 1]], 0).double()      # blocks 0, 1, 2 of the z gate
    err = float((got - ref_zr[:, :Co]).abs().max() / ref_zr[:, :Co].abs().max())
    ts = []
    for _ in range(5):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.dcrnn_bwd_wgrad(cin, K, S1, S2, dpzr, dph, True)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    res["wgmma" if tc else "ffma"] = {"us_cold": round(min(ts), 1), "rel_err_vs_fp64": err}
_lib.set_option("dcrnn_wgrad_tc", 1)
print(json.dumps(res))
