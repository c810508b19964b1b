"""Cost of the rotary position embedding (--rope) on the GPU.

    python tools/bench_rope.py [--iters 20] [--steps 10] [--blocks 8] [--images 128] [--skip_step] [--out f.json]

1. rope_fwd in place, rope_fwd out of place and rope_bwd at the ViT-10B shape (T = 32768 tokens = 128 images x 256,
   H = 32, hd = 160) and the ViT-L shape (T = 25088 = 128 x 196, H = 16, hd = 64), alternating launch by launch:
   CUDA-event time, the bytes each kernel has to move (computed from the shapes below) over that time, and that rate as
   a share of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM (a data-sheet figure, not a measured ceiling).
   Next to them, the plain qk_norm kernels against their RoPE-fused instances, alternating the same way.
2. One training step (forward_backward) of an 8-block ViT-10B at 128 images on one GPU without RoPE, with --rope, with
   --qk_norm and with --rope --qk_norm, alternating step by step, (a) with every block checkpointed and (b) with the
   automatic keep policy, plus the peak memory of each.  One model built with both flags switches them off for the other
   variants: those then run exactly the kernels of a model built without them.

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


def kernel_bytes(T, H, hd):
    """Least HBM traffic of each kernel (bf16 activations; the cos / sin tables, [N, hd / 2] fp32, stay in L2).
    rope fwd in place: read and write q, k.  Out of place: also read and copy v.  bwd: read and write dq, dk (the
    column sums are [2D]).  qk_norm: as tools/bench_qk_norm.py (read x for the backward, fp32 statistics)."""
    D = H * hd
    qk = T * 2 * D * 2
    v = T * D * 2
    stats = 2 * T * 2 * H * 4
    return {"rope_fwd_inplace": 2 * qk, "rope_fwd_out_of_place": 2 * qk + 2 * v, "rope_bwd": 2 * qk,
            "qk_norm_fwd_inplace": 2 * qk + stats, "qk_norm_rope_fwd_inplace": 2 * qk + stats,
            "qk_norm_bwd": 3 * qk + stats, "qk_norm_rope_bwd": 3 * qk + stats}


def bench_kernels(co, name, T, H, hd, grid, iters, warmup):
    from vit_10b_fsdp_example_b200.models import vit

    D, B = H * hd, T // (grid * grid)
    cos, sin = (t.cuda() for t in vit.rope_tables(grid, hd, 10000.0))
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(T, 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    scratch = qkv.clone()
    dqkv = torch.randn(T, 3 * D, device="cuda", generator=g).to(torch.bfloat16)
    w = [(torch.randn(hd, device="cuda", generator=g) * 0.1 + 1).to(torch.bfloat16) for _ in range(4)]
    rope = (cos, sin, B, 0, None)
    _, mean, rstd = co.qk_norm_fwd(qkv, H, hd, *w, 1e-5)
    rope_v = {
        # in place: each launch rotates the previous one's output, the same work every time
        "rope_fwd_inplace": (lambda: None, lambda: co.rope_fwd(scratch, H, hd, *rope, inplace=True)),
        "rope_fwd_out_of_place": (lambda: None, lambda: co.rope_fwd(qkv, H, hd, *rope)),
        "rope_bwd": (lambda: None, lambda: co.rope_bwd(dqkv, H, hd, *rope)),
    }
    qk_v = {
        "qk_norm_fwd_inplace": (lambda: None, lambda: co.qk_norm_fwd(scratch, H, hd, *w, 1e-5, inplace=True)),
        "qk_norm_rope_fwd_inplace": (lambda: None, lambda: co.qk_norm_fwd(scratch, H, hd, *w, 1e-5, inplace=True,
                                                                           rope=rope)),
        "qk_norm_bwd": (lambda: None, lambda: co.qk_norm_bwd(dqkv, qkv, H, hd, w[0], w[2], mean, rstd)),
        "qk_norm_rope_bwd": (lambda: None, lambda: co.qk_norm_bwd(dqkv, qkv, H, hd, w[0], w[2], mean, rstd,
                                                                  rope=rope)),
    }
    times = time_alternating(rope_v, iters, warmup)
    times.update(time_alternating(qk_v, iters, warmup))
    nbytes = kernel_bytes(T, H, hd)
    rec = {"shape": name, "T": T, "H": H, "hd": hd}
    for k, ts in times.items():
        ms = _med(ts)
        rec[k] = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4), "bytes": nbytes[k],
                  "tb_per_s": round(nbytes[k] / ms / 1e9, 3),
                  "share_of_3.35_datasheet": round(nbytes[k] / ms / 1e9 / HBM_TBPS, 3)}
    rec["fused_fwd_over_plain"] = round(rec["qk_norm_rope_fwd_inplace"]["ms_median"] /
                                        rec["qk_norm_fwd_inplace"]["ms_median"], 4)
    rec["fused_bwd_over_plain"] = round(rec["qk_norm_rope_bwd"]["ms_median"] / rec["qk_norm_bwd"]["ms_median"], 4)
    print(json.dumps(rec), flush=True)
    return rec


VARIANTS = {"rope_qk_norm": (True, True), "rope": (True, False), "qk_norm": (False, True), "plain": (False, False)}


def bench_step(blocks, images, steps, warmup, keep):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    torch.cuda.empty_cache()
    cfg = ViTConfig(num_blocks=blocks, rope=True, qk_norm=True)  # ViT-10B block shape: D 5120, 32 heads, 224 / 14
    model = FSDPViT(cfg, device=torch.device("cuda"), dtype=torch.bfloat16, seed=0, init_device="cuda",
                    grad_ckpt=True, ckpt_keep_blocks=keep)
    x = torch.randn(images, 3, 224, 224, device="cuda")
    y = torch.randint(0, cfg.num_classes, (images,), device="cuda")
    names = list(VARIANTS)  # the first step runs with both flags: the automatic keep policy sizes itself on its peak
    evs = {m: [] for m in names}
    peak = {m: 0 for m in names}
    losses = {m: [] for m in names}
    for i in range(len(names) * (warmup + steps)):
        m = names[i % len(names)]
        model.cfg.rope, model.cfg.qk_norm = VARIANTS[m]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        loss = model.forward_backward(x, y)
        e.record()
        torch.cuda.synchronize()
        peak[m] = max(peak[m], torch.cuda.max_memory_allocated())
        if i >= len(names) * warmup:
            evs[m].append((s, e))
            losses[m].append(loss)
    model.cfg.rope, model.cfg.qk_norm = True, True
    rec = {"step": f"forward_backward, {blocks} ViT-10B blocks, {images} images, 1 GPU, "
                   + ("all blocks checkpointed" if keep == 0 else "automatic keep policy"),
           "keep_blocks": model.keep_blocks, "keep_extras": dict(model.keep_extras)}
    for m in names:
        ts = sorted(a.elapsed_time(b) for a, b in evs[m])
        rec[m] = {"ms_median": round(_med(ts), 2), "ms_best": round(ts[0], 2),
                  "peak_mem_gib": round(peak[m] / 2 ** 30, 2), "loss_last": round(float(losses[m][-1]), 4)}
    rec["rope_over_plain"] = round(rec["rope"]["ms_median"] / rec["plain"]["ms_median"], 4)
    rec["rope_qk_norm_over_qk_norm"] = round(rec["rope_qk_norm"]["ms_median"] / rec["qk_norm"]["ms_median"], 4)
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
        sys.exit("bench_rope.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"kernels": [bench_kernels(co, "ViT-10B", 32768, 32, 160, 16, args.iters, args.warmup),
                       bench_kernels(co, "ViT-L", 25088, 16, 64, 14, args.iters, args.warmup)]}
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
