"""Time the attention core, fused kernels against the un-fused route that materialises the probabilities, without and
with attention dropout (mask drawn in registers on the fused side).

    python tools/bench_attention.py [--shapes vit10b,vitl] [--iters 20] [--warmup 3] [--p 0.1] [--out attention_bench.json]

Shapes (SHAPES): the ViT-10B and ViT-L attention, and at 128 images of 256 tokens with 16 heads the head dims of the
published larger ViTs: vith (ViT-H/14, hd 80), vitg (ViT-g/14, 88), vitG (ViT-G/14, 104), vite (ViT-e, 112) and sovit
(SoViT-400m/14, 72); hd32, hd40, hd48, hd96, hd136 and hd144 cover the other fused tile widths at the same size.
Variants, each as models/vit.py runs it for a block that keeps its activations:
  fused         attention_fwd_lse + attention_bwd_lse (no dropout)
  unfused       attention_fwd(need_p=True), which keeps P (written by the fused forward kernel), + attention_bwd (dP
                GEMM, softmax backward, three GEMMs); no dropout
  fused_drop    the same pair with drop=(p, key): Philox mask regenerated in the kernels, no [B*H, N, N] buffer
  unfused_drop  attention_fwd(drop=) (GEMM + softmax + dropout + GEMM) and, in the backward, attention_probs +
                attention_bwd(drop=) (dropout of P, dP GEMM, dropout of dP, softmax backward, three GEMMs)
Forward and backward are timed separately with CUDA events, the variants alternating launch by launch in one process;
medians over --iters.  Peak allocated bytes above the inputs are taken from one forward + backward of each variant.
The card name, power limit and SM clocks are read with a read-only nvidia-smi query before and after the run.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_gemm import gpu_info  # noqa: E402

SHAPES = {"vit10b": (128, 256, 32, 160), "vitl": (128, 196, 16, 64), "vith": (128, 256, 16, 80),
          "vitg": (128, 256, 16, 88), "vitG": (128, 256, 16, 104), "vite": (128, 256, 16, 112),
          "sovit": (128, 256, 16, 72), "hd32": (128, 256, 16, 32), "hd40": (128, 256, 16, 40),
          "hd48": (128, 256, 16, 48), "hd96": (128, 256, 16, 96), "hd136": (128, 256, 16, 136),
          "hd144": (128, 256, 16, 144)}


def variants(co, qkv, dout, B, N, H, hd, p):
    drop = (p, 0x5EED)

    def fused_fwd():
        return co.attention_fwd_lse(qkv, B, N, H, hd)

    def fused_bwd(saved):
        return co.attention_bwd_lse(dout, qkv, *saved, B, N, H, hd, want_colsum=True)

    def plain_fwd():
        return (co.attention_fwd(qkv, B, N, H, hd, need_p=True)[1],)

    def plain_bwd(saved):
        return co.attention_bwd(dout, qkv, saved[0], B, N, H, hd, want_colsum=True)

    def drop_fwd():
        return co.attention_fwd_lse(qkv, B, N, H, hd, drop=drop)

    def drop_bwd(saved):
        return co.attention_bwd_lse(dout, qkv, *saved, B, N, H, hd, want_colsum=True, drop=drop)

    def unfused_fwd():
        co.attention_fwd(qkv, B, N, H, hd, drop=drop)  # blocks do not keep P: the backward rebuilds it
        return ()

    def unfused_bwd(saved):
        P = co.attention_probs(qkv, B, N, H, hd)
        return co.attention_bwd(dout, qkv, P, B, N, H, hd, want_colsum=True, drop=drop)

    return {"fused": (fused_fwd, fused_bwd), "unfused": (plain_fwd, plain_bwd), "fused_drop": (drop_fwd, drop_bwd),
            "unfused_drop": (unfused_fwd, unfused_bwd)}


def peak_bytes(fwd, bwd):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    saved = fwd()
    bwd(saved)
    del saved
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def run_shape(co, name, B, N, H, hd, p, iters, warmup):
    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = (torch.randn(B * N, 3 * D, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda", generator=g).to(torch.bfloat16)
    vs = variants(co, qkv, dout, B, N, H, hd, p)
    peaks = {k: peak_bytes(f, b) for k, (f, b) in vs.items()}
    saved = {}
    for k, (f, b) in vs.items():
        for _ in range(warmup):
            saved[k] = f()
            b(saved[k])
    torch.cuda.synchronize()
    ev = {k: {"fwd": [], "bwd": []} for k in vs}
    for _ in range(iters):
        for k, (f, b) in vs.items():
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            s = f()
            e[1].record()
            b(s)
            e[2].record()
            ev[k]["fwd"].append((e[0], e[1]))
            ev[k]["bwd"].append((e[1], e[2]))
            del s
    torch.cuda.synchronize()
    rec = {"shape": name, "B": B, "N": N, "H": H, "hd": hd, "p": p, "iters": iters}
    for k in vs:
        fwd = sorted(a.elapsed_time(b) for a, b in ev[k]["fwd"])
        bwd = sorted(a.elapsed_time(b) for a, b in ev[k]["bwd"])
        rec[k] = {"fwd_ms_median": round(fwd[len(fwd) // 2], 4), "bwd_ms_median": round(bwd[len(bwd) // 2], 4),
                  "fwd_ms_best": round(fwd[0], 4), "bwd_ms_best": round(bwd[0], 4),
                  "peak_mib": round(peaks[k] / 2 ** 20, 1)}
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="vit10b,vitl", help="comma-separated subset of " + ",".join(SHAPES))
    ap.add_argument("--p", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="attention_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_attention.py needs a CUDA GPU")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    results = []
    for name in args.shapes.split(","):
        rec = run_shape(co, name, *SHAPES[name], args.p, args.iters, args.warmup)
        print(json.dumps(rec), flush=True)
        results.append(rec)
    summary = {"gpu_before": info_before, "gpu_after": gpu_info()}
    print(json.dumps(summary), flush=True)
    if os.path.dirname(args.out):
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"summary": summary, "shapes": results}, f, indent=1)


if __name__ == "__main__":
    main()
