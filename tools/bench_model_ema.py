"""Cost of the model EMA (--model_ema) on the GPU.

    python tools/bench_model_ema.py [--iters 30] [--steps 10] [--blocks 8] [--images 128] [--skip_step] [--out f.json]

1. adamw_split with and without the EMA operand at the shard sizes of one ViT-10B block unit for W = 1, 4 and 8,
   alternating launch by launch: CUDA-event time, the bytes each variant has to move (computed from the accesses below)
   over that time, and that rate as a share of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM (a data-sheet
   figure, not a measured ceiling).  The gradient is bf16 at W = 1 (the aliased full gradient) and fp32 at W > 1 (the
   reduce-scattered shard), as in training.
2. One training step (forward_backward + clip_grad_norm_ + AdamW) of an 8-block ViT-10B at 128 images on one GPU with
   every block checkpointed, with the EMA on and off on the same model (built with model_ema=True; the off steps pass
   no EMA operand, so they run exactly the kernels of a model without the flag), alternating step by step.
3. Peak memory of a step of that model, and of the same model built without the EMA.

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


def adamw_bytes(n, grad_bytes, ema):
    """Least HBM traffic per launch: hi, lo (2 + 2 B, read and written), m, v (4 + 4 B, read and written), the gradient
    (read); the EMA adds ema_hi + ema_lo (2 + 2 B, read and written), 8 B per element."""
    return n * (2 * (2 + 2 + 4 + 4) + grad_bytes + (8 if ema else 0))


def bench_adamw(co, W, iters, warmup):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    n = -(-ViTConfig().block_numel() // W)  # one ViT-10B block unit's shard
    gdt = torch.bfloat16 if W == 1 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(0)
    w = torch.randn(n, device="cuda", generator=g) * 0.02
    hi, lo = torch.empty(n, dtype=torch.bfloat16, device="cuda"), torch.empty(n, dtype=torch.int16, device="cuda")
    co.split_fp32(w, hi, lo)
    ehi, elo = hi.clone(), lo.clone()
    del w
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    grad = (torch.randn(n, device="cuda", generator=g) * 1e-3).to(gdt)
    hyper = torch.tensor([1e-4, 1.0], device="cuda")

    def run(ema):
        # tiny lr: every launch does the same work on almost the same values
        co.adamw_split(hi, lo, m, v, grad, None, 1e-4, 0.9, 0.999, 1e-8, 0.1, 1, hyper,
                       ema=(ehi, elo) if ema else None, ema_decay=0.9998)

    times = time_alternating({"plain": (lambda: None, lambda: run(False)), "ema": (lambda: None, lambda: run(True))},
                             iters, warmup)
    gb = torch.empty((), dtype=gdt).element_size()
    rec = {"W": W, "shard_numel": n, "grad": str(gdt).replace("torch.", "")}
    for k, ts in times.items():
        ms = _med(ts)
        nbytes = adamw_bytes(n, gb, k == "ema")
        rec[k] = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4), "bytes": nbytes,
                  "bytes_per_element": nbytes // n, "tb_per_s": round(nbytes / ms / 1e9, 3),
                  "share_of_3.35_datasheet": round(nbytes / ms / 1e9 / HBM_TBPS, 3)}
    rec["ema_over_plain"] = round(rec["ema"]["ms_median"] / rec["plain"]["ms_median"], 4)
    print(json.dumps(rec), flush=True)
    del hi, lo, ehi, elo, m, v, grad
    torch.cuda.empty_cache()
    return rec


def _step(model, opt, x, y):
    loss = model.forward_backward(x, y)
    model.clip_grad_norm_(1.0)
    opt.step()
    return loss


def bench_step(blocks, images, steps, warmup):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW

    cfg = ViTConfig(num_blocks=blocks)  # ViT-10B block shape: D 5120, 32 heads, 224 / 14
    x = torch.randn(images, 3, 224, 224, device="cuda")
    y = torch.randint(0, cfg.num_classes, (images,), device="cuda")
    torch.cuda.empty_cache()
    model = FSDPViT(cfg, device=torch.device("cuda"), dtype=torch.bfloat16, seed=0, init_device="cuda",
                    grad_ckpt=True, ckpt_keep_blocks=0, model_ema=True)
    opt = ShardedAdamW(model, lr=1e-4, weight_decay=0.1, model_ema_decay=0.9998)
    ema_bytes = sum(u.ema_hi.numel() * 2 + u.ema_lo.numel() * 2 for u in model.all_units)
    modes = (True, False)
    evs = {m: [] for m in modes}
    peak = {m: 0 for m in modes}
    for i in range(2 * (warmup + steps)):
        m = modes[i % 2]
        opt.ema_decay = 0.9998 if m else None  # None: the launches take no EMA operand
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        _step(model, opt, x, y)
        e.record()
        torch.cuda.synchronize()
        peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
        if i >= 2 * warmup:
            evs[m].append((s, e))
    rec = {"step": f"forward_backward + clip + AdamW, {blocks} ViT-10B blocks, {images} images, 1 GPU, all blocks "
                   "checkpointed", "ema_bytes": ema_bytes, "sharded_params": model.num_sharded_parameters()}
    for m in modes:
        ts = sorted(a.elapsed_time(b) for a, b in evs[m])
        rec["ema" if m else "plain"] = {"ms_median": round(_med(ts), 2), "ms_best": round(ts[0], 2),
                                        "peak_mem_gib": round(peak[m] / 2 ** 30, 2)}
    rec["ema_minus_plain_ms"] = round(rec["ema"]["ms_median"] - rec["plain"]["ms_median"], 2)
    rec["ema_over_plain"] = round(rec["ema"]["ms_median"] / rec["plain"]["ms_median"], 4)
    del model, opt
    torch.cuda.empty_cache()
    # the same model without the EMA: its peak is what a run without --model_ema needs
    model = FSDPViT(cfg, device=torch.device("cuda"), dtype=torch.bfloat16, seed=0, init_device="cuda",
                    grad_ckpt=True, ckpt_keep_blocks=0)
    opt = ShardedAdamW(model, lr=1e-4, weight_decay=0.1)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(2):
        _step(model, opt, x, y)
    torch.cuda.synchronize()
    rec["without_ema_model"] = {"peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    print(json.dumps(rec), flush=True)
    del model, opt
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--skip_step", action="store_true", help="kernels only")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_model_ema.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"adamw_split": [bench_adamw(co, W, args.iters, args.warmup) for W in (1, 4, 8)]}
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
