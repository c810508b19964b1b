"""Cost of stochastic depth (--drop_path_rate) on the GPU.

    python tools/bench_drop_path.py [--tokens 32768] [--iters 20] [--steps 20] [--blocks 8] [--images 128]
                                    [--out f.json]

1. The proj and fc2 forward GEMMs of a ViT-10B block (bias + residual epilogue) without and with the per-sample row
   scale, alternating launch by launch.
2. drop_path_bwd at [tokens, 5120]: CUDA-event time, the bytes it has to move (read dy, write dt) over that time, and
   that rate as a share of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM (a data-sheet figure, not a
   measured ceiling).
3. One training step (forward_backward) of an 8-block ViT-10B at 128 images on one GPU at rate 0 and at rate 0.2. Two
   such models (2.5 B parameters each) do not fit in 80 GB together, so one model switches its rate between steps,
   alternating 0 and 0.2.

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


def bench_gemms(co, T, D, F, N, iters, warmup):
    def r(*shape, scale=1.0):
        return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)

    B = T // N
    a, g, x = r(T, D), r(T, F, scale=0.5), r(T, D)
    w = {"proj": r(D, D, scale=0.02), "fc2": r(D, F, scale=0.02)}
    bias = {k: r(D) for k in w}
    keep = torch.rand(B, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0)) >= 0.2
    s = torch.where(keep, torch.tensor(1.25, device="cuda"), torch.tensor(0.0, device="cuda"))
    out = []
    for name, inp, K in (("proj", a, D), ("fc2", g, F)):
        variants = {
            "plain": (lambda: None, lambda inp=inp, name=name: co.linear_fwd(inp, w[name], bias[name], residual=x)),
            "row_scale": (lambda: None, lambda inp=inp, name=name: co.linear_fwd(inp, w[name], bias[name], residual=x,
                                                                                 row_scale=s, rows_per_scale=N)),
        }
        times = time_alternating(variants, iters, warmup)
        flops = 2.0 * T * D * K
        rec = {"gemm": f"{name}_fwd + bias + residual", "T": T, "N_out": D, "K": K}
        for k, ts in times.items():
            rec[k] = {"ms_median": round(_med(ts), 4), "ms_best": round(ts[0], 4),
                      "tflops_median": round(flops / _med(ts) / 1e9, 1)}
        rec["row_scale_over_plain"] = round(_med(times["row_scale"]) / _med(times["plain"]), 4)
        print(json.dumps(rec), flush=True)
        out.append(rec)
    return out


def bench_drop_path_bwd(co, T, D, N, iters, warmup):
    dy = (torch.randn(T, D, device="cuda")).to(torch.bfloat16)
    s = torch.where(torch.arange(T // N, device="cuda") % 5 == 0, 0.0, 1.25).float()
    times = time_alternating({"drop_path_bwd": (lambda: None, lambda: co.drop_path_bwd(dy, s, N))}, iters, warmup)
    ms = _med(times["drop_path_bwd"])
    nbytes = 2 * T * D * 2 + s.numel() * 4 + D * 4  # dy read, dt written, scales, column sums
    rec = {"kernel": "drop_path_bwd", "T": T, "D": D, "ms_median": round(ms, 4),
           "ms_best": round(times["drop_path_bwd"][0], 4),
           "bytes": nbytes, "tb_per_s": round(nbytes / ms / 1e9, 3),
           "share_of_3.35_datasheet": round(nbytes / ms / 1e9 / HBM_TBPS, 3)}
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
    rates = (0.0, 0.2)
    evs = {r: [] for r in rates}
    losses = {r: [] for r in rates}
    for i in range(2 * (warmup + steps)):
        r = rates[i % 2]
        model.cfg.drop_path_rate = r
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        loss = model.forward_backward(x, y)
        e.record()
        if i >= 2 * warmup:
            evs[r].append((s, e))
            losses[r].append(loss)
    torch.cuda.synchronize()
    rec = {"step": f"forward_backward, {blocks} ViT-10B blocks, {images} images, 1 GPU, all blocks checkpointed"}
    for r in rates:
        ts = sorted(a.elapsed_time(b) for a, b in evs[r])
        rec[f"rate_{r}"] = {"ms_median": round(_med(ts), 2), "ms_best": round(ts[0], 2),
                            "loss_last": round(float(losses[r][-1]), 4)}
    rec["rate_0.2_over_rate_0"] = round(rec["rate_0.2"]["ms_median"] / rec["rate_0.0"]["ms_median"], 4)
    rec["peak_mem_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 1)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=32768)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--images", type=int, default=128)
    ap.add_argument("--skip_step", action="store_true", help="kernels only")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_drop_path.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    D, N = 5120, 256
    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"gemms": bench_gemms(co, args.tokens, D, 4 * D, N, args.iters, args.warmup),
           "drop_path_bwd": bench_drop_path_bwd(co, args.tokens, D, N, args.iters, args.warmup)}
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
