"""Cost of LayerScale (--init_values) on the GPU.

    python tools/bench_layer_scale.py [--iters 20] [--steps 10] [--blocks 8] [--images 128] [--skip_step] [--out f.json]

1. layer_scale_fold and layer_scale_bwd at the ViT-10B weight shapes (proj: D 5120 x K 5120, fc2: D 5120 x K 20480),
   alternating launch by launch: CUDA-event time, the bytes each kernel has to move (computed from the shapes below)
   over that time, and that rate as a share of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM (a data-sheet
   figure, not a measured ceiling).
2. One training step (forward_backward) of an 8-block ViT-10B at 128 images on one GPU, without and with LayerScale
   (init_values 1e-5), alternating step by step, (a) with every block checkpointed and (b) with the automatic keep
   policy, plus the peak memory of each.  Two such models do not fit in 80 GB together, so one --init_values model
   switches LayerScale off for the steps without it: those run exactly the kernels of a model built without the flag.

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


def kernel_bytes(D, K):
    """Least HBM traffic of each kernel (bf16 weights; the [D] vectors are negligible).
    fold: read W, write Wg (4 B per element).  bwd: read W and M, write dW over M and Wg (8 B per element)."""
    return {"fold": 4 * D * K, "bwd": 8 * D * K}


def bench_kernels(co, name, D, K, iters, warmup):
    g = torch.Generator(device="cuda").manual_seed(0)
    W = (torch.randn(D, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    b = (torch.randn(D, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    gamma = torch.full((D,), 1e-5, device="cuda").to(torch.bfloat16)
    M = torch.randn(D, K, device="cuda", generator=g).to(torch.bfloat16)
    S = torch.randn(D, device="cuda", generator=g)
    ones = torch.ones(D, device="cuda").to(torch.bfloat16)
    variants = {
        "fold": (lambda: None, lambda: co.layer_scale_fold(W, b, gamma)),
        # in place on M with gamma = 1: every launch rewrites M with the same values, the same work every time
        "bwd": (lambda: None, lambda: co.layer_scale_bwd(W, b, ones, M, S)),
    }
    times = time_alternating(variants, iters, warmup)
    nbytes = kernel_bytes(D, K)
    rec = {"shape": name, "D": D, "K": K}
    for k, ts in times.items():
        ms = _med(ts)
        rec[k] = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4), "bytes": nbytes[k],
                  "tb_per_s": round(nbytes[k] / ms / 1e9, 3),
                  "share_of_3.35_datasheet": round(nbytes[k] / ms / 1e9 / HBM_TBPS, 3)}
    print(json.dumps(rec), flush=True)
    return rec


def bench_step(blocks, images, steps, warmup, keep, init_values=1e-5):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    torch.cuda.empty_cache()
    cfg = ViTConfig(num_blocks=blocks, init_values=init_values)  # ViT-10B block shape: D 5120, 32 heads, 224 / 14
    model = FSDPViT(cfg, device=torch.device("cuda"), dtype=torch.bfloat16, seed=0, init_device="cuda",
                    grad_ckpt=True, ckpt_keep_blocks=keep)
    x = torch.randn(images, 3, 224, 224, device="cuda")
    y = torch.randint(0, cfg.num_classes, (images,), device="cuda")
    modes = (True, False)  # the first step runs with LayerScale: the automatic keep policy sizes itself on its peak
    evs = {m: [] for m in modes}
    peak = {m: 0 for m in modes}
    losses = {m: [] for m in modes}
    for i in range(2 * (warmup + steps)):
        m = modes[i % 2]
        model.cfg.init_values = init_values if m else 0.0
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        loss = model.forward_backward(x, y)
        e.record()
        torch.cuda.synchronize()
        peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
        if i >= 2 * warmup:
            evs[m].append((s, e))
            losses[m].append(loss)
    model.cfg.init_values = init_values
    rec = {"step": f"forward_backward, {blocks} ViT-10B blocks, {images} images, 1 GPU, "
                   + ("all blocks checkpointed" if keep == 0 else "automatic keep policy"),
           "keep_blocks": model.keep_blocks, "keep_extras": dict(model.keep_extras)}
    for m in modes:
        ts = sorted(a.elapsed_time(b) for a, b in evs[m])
        rec["layer_scale" if m else "plain"] = {"ms_median": round(_med(ts), 2), "ms_best": round(ts[0], 2),
                                                "peak_mem_gib": round(peak[m] / 2 ** 30, 2),
                                                "loss_last": round(float(losses[m][-1]), 4)}
    rec["layer_scale_over_plain"] = round(rec["layer_scale"]["ms_median"] / rec["plain"]["ms_median"], 4)
    print(json.dumps(rec), flush=True)
    del model
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--skip_step", action="store_true", help="kernels only")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_layer_scale.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"kernels": [bench_kernels(co, "ViT-10B proj", 5120, 5120, args.iters, args.warmup),
                       bench_kernels(co, "ViT-10B fc2", 5120, 20480, args.iters, args.warmup)]}
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
