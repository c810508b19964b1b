"""Cost and savings of patch dropout (--patch_drop_rate) on the GPU.

    python tools/bench_patch_drop.py [--iters 20] [--steps 4] [--blocks 8] [--images 128] [--skip_step] [--out f.json]

1. The four kernels at B 128, N 256, D 5120, rate 0.5 (K 128), with P = 0 and P = 1, alternating launch by launch:
   patch_drop_select, the gathered im2col (fp32 images, patch 14), pos_gather and patch_drop_bwd.  CUDA-event time,
   the bytes each kernel has to move (computed from the shapes) over that time, and that rate as a share of the
   3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM (a data-sheet figure, not a measured ceiling).
2. One training step (forward_backward) of an 8-block ViT-10B at 128 images on one GPU at rates 0, 0.25, 0.5 and 0.75,
   without and with --class_token, plus the peak memory of each, next to the matmul-FLOP ratio computed from
   flops_per_image's formula at T'.  (a) Every block checkpointed: the rates alternate step by step on one model (the
   parameters do not depend on the rate).  (b) The automatic keep policy: it sizes itself on a variant's first step,
   so the rates run one after the other, the policy re-measured for each.

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
RATES = (0.0, 0.25, 0.5, 0.75)


def _med(ts):
    return ts[len(ts) // 2]


def kernel_bytes(B, N, K, P, D, S, ps, kpad):
    """Least HBM traffic of each kernel.  select: write keep and inv.  im2col: read the kept pixels (fp32), write the
    bf16 [B*K, kpad] columns.  pos_gather: read the [N, D] pos rows once (2.6 MB at D 5120: they stay in L2) and keep,
    write [B*K, D].  bwd: read the kept and prefix rows of dx0 and inv, write dpatch (P > 0) and the fp32 [P+N, D]
    sums."""
    return {"select": 4 * B * (K + N), "im2col": 4 * B * K * 3 * ps * ps + 2 * B * K * kpad,
            "pos_gather": 2 * B * K * D + 2 * N * D + 4 * B * K,
            "bwd": 2 * B * (P + K) * D + 4 * B * N + (2 * B * K * D if P else 0) + 4 * (P + N) * D}


def bench_kernels(co, B, N, P, D, iters, warmup):
    K, S, ps, kpad = N // 2, 224, 14, 592
    g = torch.Generator(device="cuda").manual_seed(0)
    images = torch.randn(B, 3, S, S, device="cuda", generator=g)
    pos = torch.randn(N, D, device="cuda", generator=g).to(torch.bfloat16)
    dx0 = torch.randn(B * (P + K), D, device="cuda", generator=g).to(torch.bfloat16)
    keep, inv = co.patch_drop_select(12345, B, N, K, 0, "cuda")
    variants = {
        "select": (lambda: None, lambda: co.patch_drop_select(12345, B, N, K, 0, "cuda")),
        "im2col": (lambda: None, lambda: co.patch_im2col(images, ps, kpad, torch.bfloat16, keep=keep)),
        "pos_gather": (lambda: None, lambda: co.pos_gather(pos, keep)),
        "bwd": (lambda: None, lambda: co.patch_drop_bwd(dx0, inv, B, N, K, P)),
    }
    times = time_alternating(variants, iters, warmup)
    nbytes = kernel_bytes(B, N, K, P, D, S, ps, kpad)
    rec = {"B": B, "N": N, "K": K, "P": P, "D": D}
    for k, ts in times.items():
        ms = _med(ts)
        rec[k] = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4), "ms_worst": round(ts[-1], 4),
                  "bytes": nbytes[k], "tb_per_s": round(nbytes[k] / ms / 1e9, 3),
                  "share_of_3.35_datasheet": round(nbytes[k] / ms / 1e9 / HBM_TBPS, 3)}
    print(json.dumps(rec), flush=True)
    return rec


def flop_ratio(cfg):
    """Block + stem matmul FLOPs of a training step at T' over those at T (flops_per_image's formula)."""
    D, Hd, Ho, N = cfg.embed_dim, cfg.hidden_dim, cfg.mlp_out_dim, cfg.num_patches

    def f(T, n):
        return cfg.num_blocks * (2 * T * (4 * D * D + D * Hd + D * Ho) + 4 * T * T * D) + 2 * n * cfg.patch_k * D

    return f(cfg.train_tokens, cfg.num_keep) / f(cfg.num_tokens, N)


def _timed_step(model, x, y):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    loss = model.forward_backward(x, y)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), torch.cuda.max_memory_allocated(), float(loss)


def bench_step(blocks, images, steps, warmup, class_token, auto):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    torch.cuda.empty_cache()
    dev = torch.device("cuda")
    cfgs = {r: ViTConfig(num_blocks=blocks, class_token=class_token, patch_drop_rate=r) for r in RATES}
    model = FSDPViT(cfgs[0.0], device=dev, dtype=torch.bfloat16, seed=0, init_device="cuda", grad_ckpt=True,
                    ckpt_keep_blocks=-1 if auto else 0)
    x = torch.randn(images, 3, 224, 224, device=dev)
    y = torch.randint(0, 1000, (images,), device=dev)
    res = {r: {"ms": [], "peak": 0} for r in RATES}
    if auto:  # one rate after the other, the keep policy re-sized on each rate's first step
        for r in RATES:
            model.cfg, model.keep_blocks, model._steps_here = cfgs[r], -1, 0
            for i in range(warmup + steps):
                ms, peak, loss = _timed_step(model, x, y)
                if i >= warmup:
                    res[r]["ms"].append(ms)
                    res[r]["peak"] = max(res[r]["peak"], peak)
            res[r]["keep"] = (model.keep_blocks, dict(model.keep_extras))
    else:  # alternating step by step
        for i in range(len(RATES) * (warmup + steps)):
            r = RATES[i % len(RATES)]
            model.cfg = cfgs[r]
            ms, peak, loss = _timed_step(model, x, y)
            if i >= len(RATES) * warmup:
                res[r]["ms"].append(ms)
                res[r]["peak"] = max(res[r]["peak"], peak)
    rec = {"step": f"forward_backward, {blocks} ViT-10B blocks, {images} images, 1 GPU, "
                   + ("automatic keep policy" if auto else "all blocks checkpointed"), "class_token": class_token}
    base = _med(sorted(res[0.0]["ms"]))
    for r in RATES:
        ts = sorted(res[r]["ms"])
        rec[str(r)] = {"train_tokens": cfgs[r].train_tokens, "ms_median": round(_med(ts), 2),
                       "ms_best": round(ts[0], 2), "ms_worst": round(ts[-1], 2),
                       "peak_mem_gib": round(res[r]["peak"] / 2 ** 30, 2),
                       "time_over_rate0": round(_med(ts) / base, 4), "flop_ratio": round(flop_ratio(cfgs[r]), 4)}
        if "keep" in res[r]:
            rec[str(r)]["keep_blocks"], rec[str(r)]["keep_extras"] = res[r]["keep"]
    print(json.dumps(rec), flush=True)
    del model
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--skip_step", action="store_true", help="kernels only")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_patch_drop.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"kernels": [bench_kernels(co, 128, 256, P, 5120, args.iters, args.warmup) for P in (0, 1)]}
    if not args.skip_step:
        res["step"] = [bench_step(args.blocks, args.images, args.steps, 2, ct, auto)
                       for auto in (False, True) for ct in (False, True)]
    res["gpu_before"], res["gpu_after"] = info_before, gpu_info()
    print(json.dumps({"gpu_after": res["gpu_after"]}), flush=True)
    if args.out:
        if os.path.dirname(args.out):
            os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
