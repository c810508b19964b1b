"""Cost of Mixup / CutMix / label smoothing (--mixup / --cutmix / --smoothing) on the GPU.

    python tools/bench_mixup.py [--images 128] [--iters 50] [--steps 20] [--blocks 8] [--out f.json]

1. The patch im2col at B images of 224 px, patch 14, fp32 images: plain vs Mixup vs CutMix (lam 0.3, a 112 x 112 box),
   alternating launch by launch.  The bytes are what the algorithm has to move (read every image once, write the bf16
   columns); the rate is those bytes over the kernel time, and its share of the 3.35 TB/s HBM3 data-sheet bandwidth of
   the H100 SXM (a data-sheet figure, not a measured ceiling).  Mixup reads two images per output element, so it moves
   more than that minimum unless the partner's read hits L2.
2. The cross-entropy kernel at [B, 1000]: hard labels vs the soft target of --mixup 0.8 --cutmix 1.0 --smoothing 0.1.
3. One training step (forward_backward) of an 8-block ViT-10B at B images on one GPU, with the flags at 0 and at
   --mixup 0.8 --cutmix 1.0 --smoothing 0.1, one model switching its flags between steps, alternating.

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
DEIT = dict(mixup=0.8, cutmix=1.0, smoothing=0.1)


def _med(ts):
    return ts[len(ts) // 2]


def bench_im2col(co, B, S, P, iters, warmup):
    images = torch.randn(B, 3, S, S, device="cuda")
    kpad = (3 * P * P + 7) // 8 * 8
    G = S // P
    variants = {
        "plain": (lambda: None, lambda: co.patch_im2col(images, P, kpad, torch.bfloat16)),
        "mixup": (lambda: None, lambda: co.patch_im2col(images, P, kpad, torch.bfloat16, mix=(0.3, None))),
        "cutmix": (lambda: None, lambda: co.patch_im2col(images, P, kpad, torch.bfloat16,
                                                        mix=(0.75, (56, 168, 56, 168)))),
    }
    times = time_alternating(variants, iters, warmup)
    nbytes = images.numel() * 4 + B * G * G * kpad * 2  # read the images once, write the bf16 columns
    rec = {"kernel": "im2col", "B": B, "S": S, "P": P, "image_dtype": "fp32", "bytes": nbytes}
    for k, ts in times.items():
        ms = _med(ts)
        rec[k] = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4), "tb_per_s": round(nbytes / ms / 1e9, 3),
                  "share_of_3.35_datasheet": round(nbytes / ms / 1e9 / HBM_TBPS, 3)}
    for k in ("mixup", "cutmix"):
        rec[f"{k}_over_plain"] = round(_med(times[k]) / _med(times["plain"]), 4)
    print(json.dumps(rec), flush=True)
    return rec


def bench_cross_entropy(co, B, C, iters, warmup):
    logits = (torch.randn(B, C, device="cuda") * 3).to(torch.bfloat16)
    target = torch.randint(0, C, (B,), device="cuda")
    variants = {
        "hard": (lambda: None, lambda: co.cross_entropy(logits, target)),
        "soft": (lambda: None, lambda: co.cross_entropy(logits, target, mix=(0.7, None), smoothing=0.1)),
    }
    times = time_alternating(variants, iters, warmup)
    rec = {"kernel": "cross_entropy (loss + dlogits)", "B": B, "C": C}
    for k, ts in times.items():
        rec[k] = {"ms_median": round(_med(ts), 4), "ms_best": round(ts[0], 4)}
    rec["soft_over_hard"] = round(_med(times["soft"]) / _med(times["hard"]), 4)
    print(json.dumps(rec), flush=True)
    return rec


def bench_step(blocks, images, steps, warmup):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = ViTConfig(num_blocks=blocks)  # ViT-10B block shape: D 5120, 32 heads, 224 px / patch 14
    model = FSDPViT(cfg, device=torch.device("cuda"), dtype=torch.bfloat16, seed=0, init_device="cuda",
                    grad_ckpt=True, ckpt_keep_blocks=0)
    x = torch.randn(images, 3, 224, 224, device="cuda")
    y = torch.randint(0, cfg.num_classes, (images,), device="cuda")
    settings = {"flags_0": dict(mixup=0.0, cutmix=0.0, smoothing=0.0), "deit": DEIT}
    names = list(settings)
    evs = {n: [] for n in names}
    losses = {n: [] for n in names}
    for i in range(2 * (warmup + steps)):
        n = names[i % 2]
        for k, v in settings[n].items():
            setattr(model.cfg, k, v)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        loss = model.forward_backward(x, y)
        e.record()
        if i >= 2 * warmup:
            evs[n].append((s, e))
            losses[n].append(loss)
    torch.cuda.synchronize()
    rec = {"step": f"forward_backward, {blocks} ViT-10B blocks, {images} images, 1 GPU, all blocks checkpointed"}
    for n in names:
        ts = sorted(a.elapsed_time(b) for a, b in evs[n])
        rec[n] = {"ms_median": round(_med(ts), 2), "ms_best": round(ts[0], 2),
                  "loss_last": round(float(losses[n][-1]), 4)}
    rec["deit_over_flags_0"] = round(rec["deit"]["ms_median"] / rec["flags_0"]["ms_median"], 4)
    rec["peak_mem_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--skip_step", action="store_true", help="kernels only")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mixup.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"im2col": bench_im2col(co, args.images, 224, 14, args.iters, args.warmup),
           "cross_entropy": bench_cross_entropy(co, args.images, args.classes, args.iters, args.warmup)}
    if not args.skip_step:
        res["step"] = bench_step(args.blocks, args.images, args.steps, 2)
    res["gpu_before"], res["gpu_after"] = info_before, gpu_info()
    print(json.dumps({"gpu_after": res["gpu_after"]}), flush=True)
    if args.out:
        if os.path.dirname(args.out):
            os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
