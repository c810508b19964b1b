"""Cost of the class and register tokens (--class_token / --reg_tokens) on the GPU.

    python tools/bench_prefix_tokens.py [--iters 20] [--steps 6] [--blocks 8] [--images 128] [--skip_step]
                                        [--out f.json]

1. tokens_fwd and tokens_bwd at the ViT-10B shape (B 128, N 256, D 5120) with P = 1 (T = 257) and P = 5 (T = 261),
   alternating launch by launch: CUDA-event time, the bytes each kernel has to move (computed from the shapes below)
   over that time, and that rate as a share of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM (a data-sheet
   figure, not a measured ceiling).
2. One training step (forward_backward) of an 8-block ViT-10B at 128 images on one GPU without the flags, with
   --class_token (T = 257) and with --class_token --reg_tokens 4 (T = 261), alternating step by step, (a) with every
   block checkpointed and (b) with the automatic keep policy, plus the peak memory of each.  The blocks' parameters do
   not depend on the flags and three 8-block models do not fit in 80 GB, so one model's blocks run under three root
   units (patch embed, prefix tokens, pos_embed, norm, head), swapped step by step.  The keep policy sizes itself on
   the first step, which runs with the most tokens.  At T = 257 / 261 attention takes the un-fused route (odd T), so
   the class-token steps include that route change.

Medians of --iters launches / --steps steps after warm-up, CUDA events.  The card name, its power limit and SM clocks
are read with a read-only nvidia-smi query before and after the run.
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_gemm import gpu_info, time_alternating  # noqa: E402

HBM_TBPS = 3.35  # H100 SXM HBM3, NVIDIA data sheet


def _med(ts):
    return ts[len(ts) // 2]


def kernel_bytes(B, N, P, D):
    """Least HBM traffic of each kernel (bf16 token rows, embedded prefix tokens).
    fwd: read the B*N patch rows and the P prefix and P pos rows, write the B*T token rows.
    bwd: read the B*T token-gradient rows, write the B*N patch rows and the fp32 [T, D] sums."""
    T = N + P
    return {"fwd": 2 * D * (B * N + 2 * P + B * T), "bwd": 2 * D * (B * T + B * N) + 4 * T * D}


def bench_kernels(co, B, N, P, D, iters, warmup):
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.randn(B * N, D, device="cuda", generator=g).to(torch.bfloat16)
    cls = torch.randn(1, D, device="cuda", generator=g).to(torch.bfloat16)
    reg = torch.randn(P - 1, D, device="cuda", generator=g).to(torch.bfloat16) if P > 1 else None
    pos = torch.randn(P, D, device="cuda", generator=g).to(torch.bfloat16)
    dx0 = torch.randn(B * (N + P), D, device="cuda", generator=g).to(torch.bfloat16)
    variants = {
        "fwd": (lambda: None, lambda: co.tokens_fwd(y, cls, reg, pos, B, N)),
        "bwd": (lambda: None, lambda: co.tokens_bwd(dx0, B, N, P)),
    }
    times = time_alternating(variants, iters, warmup)
    nbytes = kernel_bytes(B, N, P, D)
    rec = {"B": B, "N": N, "P": P, "T": N + P, "D": D}
    for k, ts in times.items():
        ms = _med(ts)
        rec[k] = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4), "ms_worst": round(ts[-1], 4),
                  "bytes": nbytes[k], "tb_per_s": round(nbytes[k] / ms / 1e9, 3),
                  "share_of_3.35_datasheet": round(nbytes[k] / ms / 1e9 / HBM_TBPS, 3)}
    print(json.dumps(rec), flush=True)
    return rec


VARIANTS = (("cls_reg4", dict(class_token=True, reg_tokens=4)), ("cls", dict(class_token=True)), ("plain", dict()))


def bench_step(blocks, images, steps, warmup, keep):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    torch.cuda.empty_cache()
    dev = torch.device("cuda")
    kw = dict(device=dev, dtype=torch.bfloat16, seed=0, init_device="cuda")
    model = FSDPViT(ViTConfig(num_blocks=blocks, **VARIANTS[0][1]), grad_ckpt=True, ckpt_keep_blocks=keep, **kw)
    roots = {}  # variant -> (cfg, root unit) of a block-less model: the root differs, the blocks do not
    for name, flags in VARIANTS:
        r = FSDPViT(ViTConfig(num_blocks=0, **flags), **kw)
        roots[name] = (ViTConfig(num_blocks=blocks, **flags), r.root)
    x = torch.randn(images, 3, 224, 224, device=dev)
    y = torch.randint(0, 1000, (images,), device=dev)
    names = [n for n, _ in VARIANTS]
    evs = {n: [] for n in names}
    peak = {n: 0 for n in names}
    losses = {n: [] for n in names}
    for i in range(len(names) * (warmup + steps)):
        n = names[i % len(names)]
        model.cfg, model.root = roots[n]
        model.all_units = model.units + [model.root]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        loss = model.forward_backward(x, y)
        e.record()
        torch.cuda.synchronize()
        peak[n] = max(peak[n], torch.cuda.max_memory_allocated())
        if i >= len(names) * warmup:
            evs[n].append((s, e))
            losses[n].append(loss)
    rec = {"step": f"forward_backward, {blocks} ViT-10B blocks, {images} images, 1 GPU, "
                   + ("all blocks checkpointed" if keep == 0 else "automatic keep policy"),
           "keep_blocks": model.keep_blocks, "keep_extras": dict(model.keep_extras)}
    for n in names:
        ts = sorted(a.elapsed_time(b) for a, b in evs[n])
        rec[n] = {"tokens": roots[n][0].num_tokens, "ms_median": round(_med(ts), 2), "ms_best": round(ts[0], 2),
                  "ms_worst": round(ts[-1], 2), "peak_mem_gib": round(peak[n] / 2 ** 30, 2),
                  "loss_last": round(float(losses[n][-1]), 4)}
    for n in names[:-1]:
        rec[f"{n}_over_plain"] = round(rec[n]["ms_median"] / rec["plain"]["ms_median"], 4)
    print(json.dumps(rec), flush=True)
    del model, roots
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--skip_step", action="store_true", help="kernels only")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_prefix_tokens.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"kernels": [bench_kernels(co, 128, 256, P, 5120, args.iters, args.warmup) for P in (1, 5)]}
    if not args.skip_step:
        res["step"] = [bench_step(args.blocks, args.images, args.steps, 2, keep) for keep in (0, -1)]
    res["gpu_before"], res["gpu_after"] = info_before, gpu_info()
    print(json.dumps({"gpu_after": res["gpu_after"]}), flush=True)
    if args.out:
        if os.path.dirname(args.out):
            os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
