"""Time the 12 GEMMs of one ViT block the way models/vit.py calls them (fused epilogues included) against cuBLAS.

    python tools/bench_gemm.py [--tokens 32768] [--model 10b|large] [--cluster 1,2] [--iters 10] [--out gemm_bench.json]

Per GEMM: median and best CUDA-event time, TFLOP/s, share of the 989 TFLOP/s bf16 dense data-sheet rate of the H100
SXM (a data-sheet figure, not a measured ceiling), and the bare torch.matmul (cuBLAS) GEMM of the same shape as the bar.
`--cluster 1,2` times the GEMM kernel with each CTA-cluster size (cuda_ops.set_gemm_cluster) in the same process,
alternating the variants launch by launch so that clock and power drift hit both alike.  The card name, its power
limit and SM clocks are read with a read-only nvidia-smi query before and after the run.

Every operand is far larger than the 50 MB L2 at the default size, so consecutive launches do not run from a warm L2.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_TFLOPS = 989.0  # H100 SXM, dense bf16, NVIDIA data sheet (700 W)


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, plim, cmax, csm = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(plim), "sm_max_mhz": float(cmax), "sm_mhz": float(csm)}
    except Exception as e:  # the timings stand without it; say why the card fields are missing
        return {"name": torch.cuda.get_device_name(), "nvidia_smi_error": repr(e)[:200]}


def block_gemms(co, T, D, F):
    """name -> (flops, our call, cuBLAS call).  Operand roles follow models/vit.py (forward, then backward)."""
    def r(*shape, scale=1.0):
        return (torch.randn(*shape, device="cuda") * scale).to(torch.bfloat16)

    h = r(T, D)                                     # LN output feeding qkv / fc1 (h1, h2)
    a = r(T, D)                                     # attention output feeding proj
    g = r(T, F, scale=0.5)                          # gelu(u) feeding fc2
    u = r(T, F)                                     # fc1 pre-activation
    x = r(T, D)                                     # residual stream
    w = {"qkv": r(3 * D, D, scale=0.02), "proj": r(D, D, scale=0.02), "fc1": r(F, D, scale=0.02),
         "fc2": r(D, F, scale=0.02)}
    bias = {k: r(v.shape[0]) for k, v in w.items()}
    dy_qkv, dy_d, du = r(T, 3 * D), r(T, D), r(T, F)
    gw = {k: torch.empty_like(v) for k, v in w.items()}

    def fl(m, n, k):
        return 2.0 * m * n * k

    return {
        "qkv_fwd": (fl(T, 3 * D, D), lambda: co.linear_fwd(h, w["qkv"], bias["qkv"]),
                    lambda: torch.mm(h, w["qkv"].t())),
        "proj_fwd": (fl(T, D, D), lambda: co.linear_fwd(a, w["proj"], bias["proj"], residual=x),
                     lambda: torch.mm(a, w["proj"].t())),
        "fc1_fwd": (fl(T, F, D), lambda: co.linear_fwd(h, w["fc1"], bias["fc1"], act="gelu", want_preact=True),
                    lambda: torch.mm(h, w["fc1"].t())),
        "fc2_fwd": (fl(T, D, F), lambda: co.linear_fwd(g, w["fc2"], bias["fc2"], residual=x),
                    lambda: torch.mm(g, w["fc2"].t())),
        "fc2_dgrad": (fl(T, F, D), lambda: co.linear_dgrad(dy_d, w["fc2"], dgelu_preact=u, want_colsum=True),
                      lambda: torch.mm(dy_d, w["fc2"])),
        "fc1_dgrad": (fl(T, D, F), lambda: co.linear_dgrad(du, w["fc1"]), lambda: torch.mm(du, w["fc1"])),
        "proj_dgrad": (fl(T, D, D), lambda: co.linear_dgrad(dy_d, w["proj"]), lambda: torch.mm(dy_d, w["proj"])),
        "qkv_dgrad": (fl(T, D, 3 * D), lambda: co.linear_dgrad(dy_qkv, w["qkv"]),
                      lambda: torch.mm(dy_qkv, w["qkv"])),
        "fc2_wgrad": (fl(D, F, T), lambda: co.linear_wgrad(dy_d, g, out=gw["fc2"]),
                      lambda: torch.mm(dy_d.t(), g, out=gw["fc2"])),
        "fc1_wgrad": (fl(F, D, T), lambda: co.linear_wgrad(du, h, out=gw["fc1"]),
                      lambda: torch.mm(du.t(), h, out=gw["fc1"])),
        "proj_wgrad": (fl(D, D, T), lambda: co.linear_wgrad(dy_d, a, out=gw["proj"]),
                       lambda: torch.mm(dy_d.t(), a, out=gw["proj"])),
        "qkv_wgrad": (fl(3 * D, D, T), lambda: co.linear_wgrad(dy_qkv, h, out=gw["qkv"]),
                      lambda: torch.mm(dy_qkv.t(), h, out=gw["qkv"])),
    }


def time_alternating(variants, iters, warmup):
    """variants: label -> (setup, fn).  Runs them round-robin, one launch each per round; returns label -> ms list."""
    for setup, fn in variants.values():
        setup()
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    evs = {k: [] for k in variants}
    for _ in range(iters):
        for k, (setup, fn) in variants.items():
            setup()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            evs[k].append((s, e))
    torch.cuda.synchronize()
    return {k: sorted(s.elapsed_time(e) for s, e in v) for k, v in evs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=32768)
    ap.add_argument("--model", default="10b", choices=["10b", "large"])
    ap.add_argument("--cluster", default="0", help="comma-separated CTA-cluster sizes to compare (0 = auto rule)")
    ap.add_argument("--only", default="", help="comma-separated subset of GEMM names")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="gemm_bench.json")
    args = ap.parse_args()
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    clusters = [int(c) for c in args.cluster.split(",")]
    if clusters != [0] and not hasattr(co, "set_gemm_cluster"):
        sys.exit("this build has no set_gemm_cluster: --cluster needs the clustered GEMM")
    D = 5120 if args.model == "10b" else 1024
    T, F = args.tokens, 4 * D
    info_before = gpu_info()
    gemms = block_gemms(co, T, D, F)
    if args.only:
        gemms = {k: v for k, v in gemms.items() if k in args.only.split(",")}
    results = []
    for name, (flops, ours, cublas) in gemms.items():
        variants = {}
        for c in clusters:
            setup = (lambda c=c: co.set_gemm_cluster(c)) if clusters != [0] else (lambda: None)
            variants[f"ours_c{c}"] = (setup, ours)
        variants["cublas"] = (lambda: None, cublas)
        times = time_alternating(variants, args.iters, args.warmup)
        rec = {"gemm": name, "T": T, "D": D, "tflop": flops / 1e12}
        for k, ts in times.items():
            med, best = ts[len(ts) // 2], ts[0]
            rec[k] = {"ms_median": round(med, 4), "ms_best": round(best, 4),
                      "tflops_median": round(flops / med / 1e9, 1),
                      "share_of_989_datasheet": round(flops / med / 1e9 / PEAK_TFLOPS, 3)}
        print(json.dumps(rec), flush=True)
        results.append(rec)
    if hasattr(co, "set_gemm_cluster"):
        co.set_gemm_cluster(0)
    info_after = gpu_info()
    summary = {"gpu_before": info_before, "gpu_after": info_after, "iters": args.iters,
               "sum_ms_median": {k: round(sum(r[k]["ms_median"] for r in results), 3)
                                 for k in results[0] if isinstance(results[0][k], dict)}}
    print(json.dumps(summary), flush=True)
    if os.path.dirname(args.out):
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"summary": summary, "gemms": results}, f, indent=1)


if __name__ == "__main__":
    main()
