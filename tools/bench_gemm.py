"""Time the wgmma GEMM against cuBLAS (torch.matmul) on the ViT-10B / ViT-L block shapes.

    python tools/bench_gemm.py [--tokens 32768] [--model 10b|large] [--quick] [--out gemm_bench.json]

CUDA-event timing, >= 3 warm-ups, operands far larger than L2 (or rotated) so every timed run is cold.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def time_fn(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for s, e in evs:
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) for s, e in evs)
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=32768)
    ap.add_argument("--model", default="10b")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default="gemm_bench.json")
    ap.add_argument("--block_n", type=int, default=0)
    args = ap.parse_args()
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    D = 5120 if args.model == "10b" else 1024
    T = args.tokens
    layers = [("qkv", D, 3 * D), ("proj", D, D), ("fc1", D, 4 * D), ("fc2", 4 * D, D)]
    if args.quick:
        layers = layers[:1]
    results = []
    for name, K, N in layers:
        x = torch.randn(T, K, device="cuda").to(torch.bfloat16)
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        dy = torch.randn(T, N, device="cuda").to(torch.bfloat16)
        bias = torch.randn(N, device="cuda").to(torch.bfloat16)
        flops = 2.0 * T * N * K
        cases = {
            "fwd_ours": lambda: co.linear_fwd(x, w, bias),
            "fwd_cublas": lambda: torch.nn.functional.linear(x, w, bias),
            "dgrad_ours": lambda: co.linear_dgrad(dy, w),
            "dgrad_cublas": lambda: dy @ w,
            "wgrad_ours": lambda: co.linear_wgrad(dy, x),
            "wgrad_cublas": lambda: dy.t() @ x,
        }
        if args.quick:
            cases = {k: v for k, v in cases.items() if k.startswith("fwd")}
        for cname, fn in cases.items():
            med, best = time_fn(fn, iters=5 if args.quick else 10)
            rec = {"layer": name, "case": cname, "T": T, "K": K, "N": N, "ms_median": med, "ms_best": best,
                   "tflops_median": flops / med / 1e9, "tflops_best": flops / best / 1e9}
            print(json.dumps(rec), flush=True)
            results.append(rec)
        del x, w, dy
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
