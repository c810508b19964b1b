"""Per-kernel timeline of ONE training step (CUPTI activity trace through torch.profiler -- no kernel replay, so
the step runs at its real speed with both streams and all ranks live).  Used to attribute the step-time difference
between world sizes at the same activation policy.

    python tools/step_timeline.py --blocks 8 --keep 0 --out timeline_w1.json            # 1 GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 \
        tools/step_timeline.py --blocks 8 --keep 0 --out timeline_w2.json

Per rank it reports, for the traced step: wall time (first kernel start -> last kernel end), per-stream busy time,
idle time of the compute stream, and per kernel name: launches, total / mean / max duration, stream.
"""
import argparse
import json
import os
import re
import sys
from collections import defaultdict

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def short(name: str) -> str:
    name = re.sub(r"^void\s+", "", name)
    name = re.sub(r"b200::\(anonymous namespace\)::", "", name)
    name = re.sub(r"b200::", "", name)
    name = re.sub(r"\(.*$", "", name)
    return name[:110]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--keep", type=int, default=0)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4, help="untraced timed steps (CUDA events) before the traced one")
    ap.add_argument("--model", default="vit10b")
    ap.add_argument("--device_index", type=int, default=-1)
    ap.add_argument("--backend", default="sm100", choices=["sm100", "torchdist"])
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    from bench import MODELS
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW

    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0)) if args.device_index < 0 else args.device_index
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    image, patch, dim, heads, _, mlp, _ = MODELS[args.model]
    vcfg = ViTConfig(image_size=image, patch_size=patch, embed_dim=dim, num_heads=heads, num_blocks=args.blocks,
                     mlp_ratio=mlp, num_classes=1000)
    model = FSDPViT(vcfg, world=world, rank=rank, device=dev, dtype=torch.bfloat16, backend=args.backend,
                    init_device="cuda", ckpt_keep_blocks=args.keep)
    opt = ShardedAdamW(model, lr=1e-3, weight_decay=0.1)
    x = torch.zeros(args.batch, 3, image, image, device=dev)
    y = torch.zeros(args.batch, dtype=torch.long, device=dev)

    def step():
        model.forward_backward(x, y)
        model.clip_grad_norm_(1.0)
        opt.step()
        opt.zero_grad()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    untraced_ms = e0.elapsed_time(e1) / max(1, args.steps)

    from torch.profiler import ProfilerActivity, profile

    if world > 1:
        dist.barrier()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    kin = prof.profiler.kineto_results.events()
    rows = []
    for e in kin:
        if "cuda" not in str(e.device_type()).lower():
            continue
        nm = e.name()
        if nm.startswith("Memcpy") or nm.startswith("Memset"):
            nm = nm.split(" ")[0]
        rows.append((short(nm), int(e.device_resource_id()), e.start_ns() / 1e3, e.duration_ns() / 1e3))
    if not rows:
        print(f"[rank {rank}] no CUDA activity records captured", flush=True)
        return
    t0 = min(r[2] for r in rows)
    t1 = max(r[2] + r[3] for r in rows)
    per_stream = defaultdict(float)
    agg = defaultdict(lambda: [0, 0.0, 0.0, set()])
    for nm, st, s, d in rows:
        per_stream[st] += d
        a = agg[nm]
        a[0] += 1
        a[1] += d
        a[2] = max(a[2], d)
        a[3].add(st)
    main_stream = max(per_stream, key=per_stream.get)
    # union of busy intervals on the compute stream (kernels on one stream do not overlap, but be safe)
    iv = sorted((s, s + d) for nm, st, s, d in rows if st == main_stream)
    busy, cur_s, cur_e = 0.0, None, None
    gaps = []
    for s, e in iv:
        if cur_e is None:
            cur_s, cur_e = s, e
        elif s <= cur_e:
            cur_e = max(cur_e, e)
        else:
            gaps.append((s - cur_e, cur_e - t0))
            busy += cur_e - cur_s
            cur_s, cur_e = s, e
    busy += cur_e - cur_s
    gaps.sort(reverse=True)
    res = {
        "rank": rank, "world": world, "blocks": args.blocks, "keep": args.keep, "batch": args.batch,
        "untraced_ms_per_step": untraced_ms, "traced_wall_ms": (t1 - t0) / 1e3,
        "compute_stream": main_stream, "compute_busy_ms": busy / 1e3, "compute_idle_ms": (t1 - t0 - busy) / 1e3,
        "stream_busy_ms": {str(k): v / 1e3 for k, v in per_stream.items()},
        "largest_gaps_us_at_ms": [(round(g, 1), round(at / 1e3, 2)) for g, at in gaps[:12]],
        "kernels": sorted(({"name": k, "n": v[0], "total_ms": v[1] / 1e3, "mean_us": v[1] / v[0], "max_us": v[2],
                            "streams": sorted(v[3])} for k, v in agg.items()), key=lambda r: -r["total_ms"]),
    }
    gpu = torch.cuda.get_device_name(dev)
    print(f"[rank {rank}/{world} {gpu} dev{local}] untraced {untraced_ms:.1f} ms/step  traced wall "
          f"{res['traced_wall_ms']:.1f}  compute busy {res['compute_busy_ms']:.1f}  idle {res['compute_idle_ms']:.1f}",
          flush=True)
    for r in res["kernels"][:28]:
        print(f"   r{rank} {r['total_ms']:9.2f} ms  n={r['n']:4d}  mean {r['mean_us']:9.1f} us  max {r['max_us']:9.1f}  "
              f"s={r['streams']}  {r['name'][:90]}", flush=True)
    if args.out:
        path = args.out.replace(".json", f"_r{rank}.json")
        with open(path, "w") as f:
            json.dump(res, f, indent=1)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
