"""Cost of the SwiGLU MLP (--swiglu) on the GPU.

    python tools/bench_swiglu.py [--iters 20] [--tokens 32768] [--steps 6] [--blocks 4] [--images 64] [--skip_step]
                                 [--out f.json]

At two shapes, ViT-10B class (D 5120, SwiGLU Hd 27296, GELU Hd 20480: the same MLP parameter count to 0.04 %) and
DINOv2-g (D 1536, SwiGLU Hd 8192, GELU Hd 6144), with --tokens rows, alternating launch by launch:
1. fc1 forward + SwiGLU: the fused epilogue without and with the pre-activation side output, against the plain GEMM
   (which writes u) + swiglu_fwd, and the fused GELU epilogue of the GELU MLP with the same parameter count.
2. fc2 dgrad + dSwiGLU + the fc1 bias column sums: fused against the plain dgrad + swiglu_bwd + colsum, and the fused
   dGELU dgrad of the GELU MLP.
3. swiglu_fwd / swiglu_bwd alone: the bytes they must move over their time, as a share of the 3.35 TB/s HBM3
   data-sheet bandwidth of the H100 SXM (a data-sheet figure, not a measured ceiling).
4. One training step (forward_backward) of a reduced-depth ViT-10B on one GPU, GELU MLP (mlp_ratio 4) against SwiGLU
   (Hd 27296) at the same parameter count, every block checkpointed, alternating step by step.

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
SHAPES = {"ViT-10B class": (5120, 27296, 20480), "DINOv2-g": (1536, 8192, 6144)}  # D, SwiGLU Hd, GELU Hd


def _med(ts):
    return ts[len(ts) // 2]


def _rec(ts, flops=None, nbytes=None):
    ms = _med(ts)
    r = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4)}
    if flops:
        r["tflop_per_s"] = round(flops / ms / 1e9, 1)
    if nbytes:
        r["tb_per_s"] = round(nbytes / ms / 1e9, 3)
        r["share_of_3.35_datasheet"] = round(nbytes / ms / 1e9 / HBM_TBPS, 3)
    return r


def bench_gemms(co, name, T, D, Hd, Hg, iters, warmup):
    def r(*shape, scale=1.0):
        return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)

    Hh = Hd // 2
    h, w1, b1, wg, bg = r(T, D), r(Hd, D, scale=0.02), r(Hd, scale=0.02), r(Hg, D, scale=0.02), r(Hg, scale=0.02)
    dt, w2, w2g = r(T, D), r(D, Hh, scale=0.02), r(D, Hg, scale=0.02)
    u, ug = co.linear_fwd(h, w1, b1), co.linear_fwd(h, wg, bg)
    old = co.FUSE_ACT_MIN_K, co.SWIGLU_FWD_MIN_K, co.SWIGLU_DGRAD_K
    # the fused epilogues at every K; the unfused variants call the plain pieces directly
    co.FUSE_ACT_MIN_K, co.SWIGLU_FWD_MIN_K, co.SWIGLU_DGRAD_K = 0, 0, (0, 1 << 30)
    try:
        fwd = {
            "swiglu_fused": (lambda: None, lambda: co.linear_fwd(h, w1, b1, act="swiglu")),
            "swiglu_fused_preact": (lambda: None, lambda: co.linear_fwd(h, w1, b1, act="swiglu", want_preact=True)),
            "swiglu_unfused": (lambda: None, lambda: co.swiglu_fwd(co.linear_fwd(h, w1, b1))),
            "gelu_fused_preact": (lambda: None, lambda: co.linear_fwd(h, wg, bg, act="gelu", want_preact=True)),
        }
        bwd = {
            "dswiglu_fused": (lambda: None, lambda: co.linear_dgrad(dt, w2, dswiglu_preact=u, want_colsum=True)),
            "dswiglu_unfused": (lambda: None, lambda: co.colsum(co.swiglu_bwd(co.linear_dgrad(dt, w2), u))),
            "dgelu_fused": (lambda: None, lambda: co.linear_dgrad(dt, w2g, dgelu_preact=ug, want_colsum=True)),
        }
        tf, tb = time_alternating(fwd, iters, warmup), time_alternating(bwd, iters, warmup)
    finally:
        co.FUSE_ACT_MIN_K, co.SWIGLU_FWD_MIN_K, co.SWIGLU_DGRAD_K = old
    ff = {k: 2 * T * D * (Hg if k.startswith("gelu") else Hd) for k in fwd}
    fb = {k: 2 * T * D * (Hg if k.startswith("dgelu") else Hh) for k in bwd}
    rec = {"shape": name, "T": T, "D": D, "Hd_swiglu": Hd, "Hd_gelu": Hg,
           "fc1_forward": {k: _rec(v, ff[k]) for k, v in tf.items()},
           "fc2_dgrad": {k: _rec(v, fb[k]) for k, v in tb.items()}}
    f, b = rec["fc1_forward"], rec["fc2_dgrad"]
    rec["fused_over_unfused"] = {"forward_preact": round(f["swiglu_fused_preact"]["ms_median"]
                                                         / f["swiglu_unfused"]["ms_median"], 3),
                                 "dgrad": round(b["dswiglu_fused"]["ms_median"] / b["dswiglu_unfused"]["ms_median"], 3)}
    g = torch.Generator(device="cuda").manual_seed(0)
    dg = torch.randn(T, Hh, device="cuda", generator=g).to(torch.bfloat16)
    tm = time_alternating({"swiglu_fwd": (lambda: None, lambda: co.swiglu_fwd(u)),
                           "swiglu_bwd": (lambda: None, lambda: co.swiglu_bwd(dg, u))}, iters, warmup)
    # least HBM traffic: fwd reads u [T, Hd] and writes g [T, Hd/2]; bwd reads dg and u and writes du [T, Hd]
    rec["memory_bound"] = {"swiglu_fwd": _rec(tm["swiglu_fwd"], nbytes=3 * T * Hd),
                           "swiglu_bwd": _rec(tm["swiglu_bwd"], nbytes=5 * T * Hd)}
    print(json.dumps(rec), flush=True)
    return rec


def bench_step(blocks, images, steps, warmup):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    torch.cuda.empty_cache()
    cfgs = {"gelu": ViTConfig(num_blocks=blocks),
            "swiglu": ViTConfig(num_blocks=blocks, swiglu=True, mlp_ratio=(27296 + 0.5) / 5120)}
    assert cfgs["swiglu"].hidden_dim == 27296
    models = {k: FSDPViT(c, device=torch.device("cuda"), dtype=torch.bfloat16, seed=0, init_device="cuda",
                         grad_ckpt=True, ckpt_keep_blocks=0) for k, c in cfgs.items()}
    x = torch.randn(images, 3, 224, 224, device="cuda")
    y = torch.randint(0, 1000, (images,), device="cuda")
    evs = {k: [] for k in models}
    for i in range(warmup + steps):
        for k, m in models.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            m.forward_backward(x, y)
            e.record()
            torch.cuda.synchronize()
            if i >= warmup:
                evs[k].append((s, e))
    rec = {"step": f"forward_backward, {blocks} ViT-10B blocks, {images} images, 1 GPU, all blocks checkpointed",
           "params": {k: m.num_parameters() for k, m in models.items()},
           "flops_per_image": {k: c.flops_per_image() for k, c in cfgs.items()}}
    for k in models:
        rec[k] = _rec(sorted(a.elapsed_time(b) for a, b in evs[k]))
    rec["swiglu_over_gelu"] = round(rec["swiglu"]["ms_median"] / rec["gelu"]["ms_median"], 4)
    print(json.dumps(rec), flush=True)
    del models
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tokens", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--skip_step", action="store_true", help="kernels only")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_swiglu.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"gemms": [bench_gemms(co, name, args.tokens, *s, args.iters, args.warmup) for name, s in SHAPES.items()]}
    torch.cuda.empty_cache()
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
