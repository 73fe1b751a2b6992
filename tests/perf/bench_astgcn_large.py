"""ASTGCN inference on the PeMS03 / PeMS07 shapes (358 / 883 nodes): the cfg4 architecture ASTGCN(3 blocks, K=3, 64/64 filters, 12 -> 12),
B = 32 windows, no_grad, on the native channels-last path (column-tiled spatial attention, csrc/spatial_attention_tiled.cu) against the
op-for-op path (forced here by turning the blocks' native gate off).  Also the spatial-attention pair alone (k_spatt_tiles + k_spatt_norm)
with its fp16-split tensor FLOPs (3 passes x 2 B N Npad^2) and the bytes of ST it writes and re-reads.  CUDA events; the paths are
alternated, three runs each.  Prints the card and its power limit (read in the same run) and one JSON line per shape.
    python tests/perf/bench_astgcn_large.py [--steps N] [--shapes pems03,pems07]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--shapes", default="pems03,pems07")
args = ap.parse_args()

import torch  # noqa: E402

from pytorch_geometric_temporal_b200 import ops  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN  # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import astgcn as astgcn_mod  # noqa: E402

DEV = "cuda"
B, T = 32, 12
SHAPES = {"pems03": (synthetic.pems03_like, 358), "pems07": (synthetic.pems07_like, 883)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        pl, clk = float(q[0]), float(q[1])
    except (OSError, subprocess.SubprocessError, ValueError, IndexError):
        pl = clk = None
    return torch.cuda.get_device_name(), pl, clk


def timed(fn, steps):
    """ms per call from CUDA events around `steps` calls, after two warm-up calls"""
    for _ in range(2):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def alternate(fns, steps):
    res = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            res[k].append(round(timed(fn, steps), 4))
    return res


NATIVE_OK = astgcn_mod.ASTGCNBlock._native_ok


def forward(m, X, ei, native):
    def f():
        astgcn_mod.ASTGCNBlock._native_ok = NATIVE_OK if native else (lambda self, N, Fi, T: False)
        try:
            with torch.no_grad():
                return m(X, ei)
        finally:
            astgcn_mod.ASTGCNBlock._native_ok = NATIVE_OK
    return f


def main():
    gpu, pl, clk = card()
    print(json.dumps({"bench": "astgcn_large", "gpu": gpu, "power_limit_w": pl, "max_sm_clock_mhz": clk}), flush=True)
    for name in args.shapes.split(","):
        like, n = SHAPES[name]
        ei = torch.from_numpy(like(0)).to(DEV)
        torch.manual_seed(0)
        m = ASTGCN(3, 1, 3, 64, 64, 1, 12, 12, n, normalization="sym").to(DEV)
        X = torch.randn(B, n, 1, T, device=DEV)
        fwd = alternate({"native": forward(m, X, ei, True), "op_for_op": forward(m, X, ei, False)}, args.steps)
        out_n, out_t = forward(m, X, ei, True)(), forward(m, X, ei, False)()
        # the spatial-attention pair alone, on the first block's factors
        blk = m._blocklist[0]
        ta, sa = blk._temporal_attention, blk._spatial_attention
        with torch.no_grad():
            lhs, rhs = ops.astgcn_factors(X.permute(0, 1, 3, 2).contiguous(), ta._U1, ta._U2, ta._U3, ta._be, ta._Ve, sa._W1, sa._W2, sa._W3)
            pk = blk._native_packs()
        P = (n + 63) // 64 * 64
        spatt = alternate({"spatt": lambda: ops.spatial_attention(lhs, rhs, pk["bsT"], pk["vsT"])}, 5 * args.steps)["spatt"]
        flops = 3 * 2 * B * n * P * P
        st_bytes = 3 * B * n * P * 4                      # logits written, read and rewritten by the normalisation
        best = min(spatt)
        print(json.dumps({"shape": name, "nodes": n, "edges": int(ei.size(1)), "B": B, "T": T, "forward_ms": fwd,
                          "native_vs_op_for_op_max_abs_diff": (out_n - out_t).abs().max().item(),
                          "spatt_ms": spatt, "spatt_tensor_tflops": round(flops / best / 1e9, 1), "spatt_st_gb_per_s": round(st_bytes / best / 1e6, 1),
                          "spatt_flops": flops, "spatt_st_bytes": st_bytes}), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
