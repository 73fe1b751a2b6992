#!/usr/bin/env python
"""BASELINE configs[3] on N GPUs: ASTGCN(3 blocks, K=3, 64/64 filters, 12 -> 12) on the synthetic PeMS04 shape (307 nodes, 340 links),
batch 32 per GPU, data-parallel.

  python tests/perf/bench_cfg4_ddp.py                                                       (1 GPU)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 --master-port 29512 tests/perf/bench_cfg4_ddp.py

Two numbers (rank 0 prints one JSON line; device-timed, max over ranks):
  * inference: windows/s through the native channels-last path (fused spatial attention + blocked wgmma GEMMs), replicas, no collective;
  * training:  windows/s of forward + backward (autograd around stmp_spmm / stmp_spmm_att_grad) + ONE flat NCCL all-reduce + Adam."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from pytorch_geometric_temporal_b200 import _lib, distributed as D           # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic                # noqa: E402
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN              # noqa: E402


def timed(fn, steps, warmup, world, dev):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item()) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    rank, world, dev = D.init_process_group()
    ei = torch.from_numpy(synthetic.pems04_like(0)).to(dev)
    torch.manual_seed(0)
    m = ASTGCN(3, 1, 3, 64, 64, 1, 12, 12, 307, normalization="sym").to(dev)
    if world > 1:
        D.broadcast_parameters(m)
    g = torch.Generator(device=dev).manual_seed(100 + rank)
    X = torch.randn(args.batch, 307, 1, 12, device=dev, generator=g)
    Y = torch.randn(args.batch, 307, 12, device=dev, generator=g)

    def infer():
        with torch.no_grad():
            return m(X, ei)
    ms_inf = timed(infer, args.steps, args.warmup, world, dev)
    sync = D.FlatGradSync(m.parameters())
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)

    def train():
        loss = torch.nn.functional.l1_loss(m(X, ei), Y)
        loss.backward()
        sync.all_reduce()
        opt.step()
        sync.zero()
    ms_tr = timed(train, max(3, args.steps // 2), 3, world, dev)
    if rank == 0:
        pc = {k: v for k, v in _lib.path_counters().items() if v and k in ("k_gemm_blocks", "k_astgcn_factors", "k_spmm", "k_att_grad")}
        print(json.dumps({"config": "cfg4 ASTGCN(3 blocks,K=3,64/64) PeMS04 shape (307 nodes), batch 32 per GPU, data-parallel", "n_gpus": world,
                          "inference_ms_per_step": ms_inf, "inference_windows_per_s": world * args.batch / (ms_inf * 1e-3),
                          "training_ms_per_step": ms_tr, "training_windows_per_s": world * args.batch / (ms_tr * 1e-3),
                          "allreduce_bytes_per_step": sync.nbytes if world > 1 else 0, "kernels": pc}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
