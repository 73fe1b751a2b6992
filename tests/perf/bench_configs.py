#!/usr/bin/env python
"""(lives under tests/: it times the oracle as the CPU side, and only tests/, smoke() and bench.py may touch oracle/)
Secondary measurements for the other BASELINE.json configs (parity-test cases, not bench lines):
cfg1 GConvGRU/chickenpox, cfg3 A3TGCN2/PEMS-BAY-shape, cfg4 ASTGCN/PeMS04-shape, cfg5 GConvLSTM 10k/100k.
Prints one JSON object per config: ours (CUDA events, after warm-up) and the oracle port on the host cores."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import attention as OA, recurrent as R  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import ChickenpoxDatasetLoader, synthetic  # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN  # noqa: E402
from pytorch_geometric_temporal_b200.nn.recurrent import A3TGCN2, GConvGRU, GConvLSTM  # noqa: E402

DEV = torch.device("cuda")


def gpu_time(fn, iters=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def cpu_time(fn, budget=6.0, threads=16):
    torch.set_num_threads(min(threads, os.cpu_count() or 1))
    fn()
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < budget:
        fn(); n += 1
    return (time.perf_counter() - t0) / n * 1e3


def graphed(fn):
    """Replay a fixed launch sequence from a CUDA graph (falls back to eager)."""
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                fn()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        return g.replay, "cuda-graph"
    except Exception as e:  # noqa
        torch.cuda.synchronize()
        return fn, f"eager ({type(e).__name__})"


def main():
    out = []
    with torch.no_grad():
        # cfg1 -------------------------------------------------------------------------------------------------
        ds = ChickenpoxDatasetLoader().get_dataset(lags=4)
        snaps = [ds[t] for t in range(64)]
        torch.manual_seed(0)
        m = GConvGRU(4, 32, 2); sd = m.state_dict(); mg = m.to(DEV)
        gs = [s.to(DEV) for s in snaps]
        def ours():
            H = None
            for s in gs:
                H = mg(s.x, s.edge_index, s.edge_attr, H)
        def cpu():
            H = None
            for s in snaps:
                H = R.gconv_gru_cell(sd, s.x, s.edge_index, s.edge_attr, H)
        run, how = graphed(ours)
        ms, cms = gpu_time(run), cpu_time(cpu)
        out.append({"config": "cfg1 GConvGRU(4,32,K=2) chickenpox (20 nodes), 64 chained snapshots", "launch": how, "ours_ms": ms,
                    "ours_snapshots_per_s": 64 / ms * 1e3, "cpu_oracle_ms": cms, "cpu_snapshots_per_s": 64 / cms * 1e3})
        # cfg3 -------------------------------------------------------------------------------------------------
        ei, ew, _ = synthetic.pems_bay_like(0, 16)
        ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
        torch.manual_seed(0)
        m = A3TGCN2(2, 32, 12, 64); sd = m.state_dict(); head = torch.nn.Linear(32, 12)
        X = torch.randn(64, 325, 2, 12)
        mg, hg, Xg, eig, ewg = m.to(DEV), head.to(DEV), X.to(DEV), ei.to(DEV), ew.to(DEV)
        run, how = graphed(lambda: hg(torch.relu(mg(Xg, eig, ewg))))
        ms = gpu_time(run)
        cms = cpu_time(lambda: R.a3tgcn(sd, X[:8], ei, ew)) * 8  # 8 of 64 batch rows, scaled
        out.append({"config": "cfg3 A3TGCN2(2,32,12 periods)+Linear, PEMS-BAY shape (325 nodes), batch 64", "launch": how, "ours_ms": ms,
                    "ours_batches_per_s": 1e3 / ms, "cpu_oracle_ms_scaled_from_8_rows": cms, "cpu_batches_per_s": 1e3 / cms})
        # cfg4 -------------------------------------------------------------------------------------------------
        eiu = torch.from_numpy(synthetic.pems04_like(0))
        torch.manual_seed(0)
        m = ASTGCN(3, 1, 3, 64, 64, 1, 12, 12, 307, normalization="sym"); sd = m.state_dict()
        X = torch.randn(32, 307, 1, 12)
        mg, Xg, eg = m.to(DEV), X.to(DEV), eiu.to(DEV)
        run, how = graphed(lambda: mg(Xg, eg))
        ms = gpu_time(run)
        cms = cpu_time(lambda: OA.astgcn(sd, X[:4], eiu, 3, "sym", 1), budget=8) * 8
        out.append({"config": "cfg4 ASTGCN(3 blocks,K=3,64/64) PeMS04 shape (307 nodes), batch 32, forward", "launch": how, "ours_ms": ms,
                    "ours_windows_per_s": 32 / ms * 1e3, "cpu_oracle_ms_scaled_from_4_rows": cms, "cpu_windows_per_s": 32 / cms * 1e3})
        # cfg5 -------------------------------------------------------------------------------------------------
        ei, ew = synthetic.large_graph(10000, 100000, 0)
        ei, ew = torch.from_numpy(ei), torch.from_numpy(ew)
        torch.manual_seed(0)
        m = GConvLSTM(64, 64, 3); sd = m.state_dict()
        X = torch.randn(8, 12, 10000, 64)
        mg, Xg, eig, ewg = m.to(DEV), X.to(DEV), ei.to(DEV), ew.to(DEV)
        def ours5():
            H = C = None
            for t in range(12):
                H, C = mg(Xg[:, t], eig, ewg, H, C)
        def cpu5():
            H = C = None
            for t in range(2):
                H, C = R.gconv_lstm_cell(sd, X[0, t], ei, ew, H, C)
        run, how = graphed(ours5)
        ms = gpu_time(run, iters=10)
        cms = cpu_time(cpu5, budget=8) * 6 * 8  # 2 of 12 steps, 1 of 8 windows, scaled
        out.append({"config": "cfg5 GConvLSTM(64,64,K=3), 10k nodes / 100k edges, 8 windows x 12 steps per GPU, forward", "launch": how,
                    "ours_ms": ms, "ours_snapshots_per_s": 8 / ms * 1e3, "cpu_oracle_ms_scaled": cms, "cpu_snapshots_per_s": 8 / cms * 1e3})
        # K4 probe: the wgmma split-fp16 GEMM alone at the cfg5 size, vs cuBLAS fp32 (torch.matmul)
        from pytorch_geometric_temporal_b200 import ops
        A = torch.randn(80000, 384, device=DEV); W = torch.randn(384, 256, device=DEV) * 0.1
        packed = ops.gemm_prepack(W)
        ms_tc = gpu_time(lambda: ops.gemm(A, packed, 384, 256), iters=20)
        ms_cb = gpu_time(lambda: torch.matmul(A, W), iters=20)
        byt = 80000 * 384 * 4 + 80000 * 256 * 4
        pk_b = ops.gemm_blocks_prepack([W[64 * i:64 * i + 64].contiguous() for i in range(6)])
        Cb = torch.empty(80000, 256, device=DEV)
        ms_gb = gpu_time(lambda: ops.gemm_blocks([(A[:, 64 * i:64 * i + 64], 64, 0) for i in range(6)], pk_b, 256, 256, None, ops.EPI_BIAS, out=Cb), iters=20)
        out.append({"config": "K4 probe: C[80000,256] = A[80000,384] @ W, fp32 in/out", "wgmma_split_fp16_ms": ms_tc, "cublas_fp32_ms": ms_cb,
                    "wgmma_blocked_ms (TMA weight image, prefetched A)": ms_gb,
                    "algorithmic_bytes": byt, "achieved_gbs": byt / ms_tc / 1e6, "blocked_achieved_gbs": byt / ms_gb / 1e6,
                    "tflops_fp32_equiv": 2 * 80000 * 384 * 256 / ms_tc / 1e9})
    for o in out:
        print(json.dumps(o))


if __name__ == "__main__":
    main()
