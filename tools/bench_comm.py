"""Collective micro-benchmark: the hand-written symmetric-memory all-gather / reduce-scatter kernels (csrc/comm.cu)
against NCCL for the message sizes of the ViT configs (3 MiB ... 600 MiB of bf16 per unit).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 \
        tools/bench_comm.py [--out bench_comm.json]

Times are CUDA-event medians on the launching stream, max over ranks.  "bus GB/s" is the per-GPU ingress
(W-1)/W * bytes / time, the figure to hold against the NVLink line rate of an H100 SXM (450 GB/s per direction); with
NVLS the reduce-scatter ingress is 1/W of that (the switch reduces), so its number is reported as algorithm bandwidth.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vit_10b_fsdp_example_b200.ops import cuda_ops  # noqa: E402
from vit_10b_fsdp_example_b200.parallel.backends import Sm100Backend  # noqa: E402
from vit_10b_fsdp_example_b200.parallel.layout import UnitLayout  # noqa: E402


def timed(fn, iters=20, warm=5):
    for _ in range(warm):
        fn()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    torch.cuda.synchronize()
    dist.barrier()
    for a, b in evs:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in evs)[iters // 2]
    t = torch.tensor([ms], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    be = Sm100Backend(world, rank, dev)
    rows = []
    for mib in (3, 18, 75, 150, 300, 600):  # full (gathered) size of one unit in bf16
        cols = 4096
        nrow = max(world * 8, (mib * 2 ** 20 // 2 // cols) // (world * 8) * (world * 8))
        lay = UnitLayout.build("u", [("w", (nrow, cols))], world, False)
        shard = be.alloc_shard(lay.shard_numel, torch.bfloat16)
        shard.normal_()
        full = torch.empty(lay.full_numel, dtype=torch.bfloat16, device=dev)
        grad = be.alloc_full_grad(lay.full_numel, torch.bfloat16)
        grad.normal_()
        out32 = torch.empty(lay.shard_numel, dtype=torch.float32, device=dev)
        sumsq = torch.zeros(1, device=dev)
        be.params_updated()
        nbytes = lay.full_numel * 2
        ingress = nbytes * (world - 1) / world
        full_nccl = torch.empty(world * lay.shard_numel, dtype=torch.bfloat16, device=dev)
        grad32 = grad.float()
        out_nccl = torch.empty(lay.shard_numel, dtype=torch.float32, device=dev)
        r = {"world": world, "full_MiB": nbytes / 2 ** 20, "nvls": bool(be.use_nvls)}
        for transport in ("kernel", "ce"):  # light pull kernel vs copy engines
            be.ag_transport = transport
            full.zero_()
            t = timed(lambda: be.all_gather(lay, shard, full))
            r[f"ag_{transport}_ms"], r[f"ag_{transport}_busGBs"] = t, ingress / t / 1e6
            dist.all_gather_into_tensor(full_nccl, shard)
            torch.cuda.synchronize()
            r[f"ag_{transport}_exact"] = bool(torch.equal(full.view(world, -1), full_nccl.view(world, -1)))
        t = timed(lambda: dist.all_gather_into_tensor(full_nccl, shard))
        r["ag_nccl_ms"], r["ag_nccl_busGBs"] = t, ingress / t / 1e6
        t = timed(lambda: be.reduce_scatter(lay, grad, out32, sumsq, cuda_ops))
        r["rs_custom_ms"], r["rs_custom_algGBs"] = t, nbytes / t / 1e6
        t = timed(lambda: dist.reduce_scatter_tensor(out_nccl, grad32, op=dist.ReduceOp.AVG))
        r["rs_nccl_fp32_ms"], r["rs_nccl_fp32_algGBs"] = t, nbytes * 2 / t / 1e6
        rows.append(r)
        if rank == 0:
            print(json.dumps(r), flush=True)
        del shard, full, grad, out32, full_nccl, grad32, out_nccl
    if rank == 0 and args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
