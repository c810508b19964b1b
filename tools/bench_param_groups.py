"""Cost of the optimizer parameter groups (--filter_bias_and_norm / --layer_decay) in the AdamW kernels, on the GPU.

    python tools/bench_param_groups.py [--iters 50] [--warmup 5] [--out f.json]

The grouped adamw_split against the plain one, with and without the EMA operand, at the shard lengths of the ViT-10B
block unit and root unit for W = 4 and 8 (fp32 reduce-scattered gradient, as in training at W > 1).  The group tables
are the real ones of rank 0 (parallel/param_groups.py, layer decay 0.75).  The four variants run round-robin, one
launch each per round.  Reported per variant: median and best CUDA-event time, the bytes the kernel must move (computed
from its accesses below) over the median time, and that rate as a share of the 3.35 TB/s HBM3 data-sheet bandwidth of the
H100 SXM (a data-sheet figure, not a measured ceiling).  The card name, power limit and SM clocks are read with a
read-only nvidia-smi query before and after the run.
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


def adamw_bytes(n, grad_bytes, ema, grouped):
    """Least HBM traffic per launch: hi, lo (2 + 2 B, read and written), m, v (4 + 4 B, read and written), the gradient
    (read); the EMA adds ema_hi + ema_lo (2 + 2 B, read and written); the groups add one uint8 per 64 elements."""
    return n * (2 * (2 + 2 + 4 + 4) + grad_bytes + (8 if ema else 0)) + (n // 64 if grouped else 0)


def bench_unit(co, unit, W, iters, warmup):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.models import vit
    from vit_10b_fsdp_example_b200.parallel import param_groups as pg
    from vit_10b_fsdp_example_b200.parallel.layout import UnitLayout

    cfg = ViTConfig()
    specs = vit.root_param_specs(cfg) if unit == "root" else vit.block_param_specs(cfg)
    lay = UnitLayout.build("root" if unit == "root" else "blocks.0", specs, W, False)
    ug = pg.build_unit_groups(cfg, lay, 0, 0.1, 0.75, "cuda")
    n = lay.shard_numel
    g = torch.Generator(device="cuda").manual_seed(0)
    w = torch.randn(n, device="cuda", generator=g) * 0.02
    hi, lo = torch.empty(n, dtype=torch.bfloat16, device="cuda"), torch.empty(n, dtype=torch.int16, device="cuda")
    co.split_fp32(w, hi, lo)
    ehi, elo = hi.clone(), lo.clone()
    del w
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    grad = torch.randn(n, device="cuda", generator=g) * 1e-3
    hyper = torch.tensor([1e-4, 1.0], device="cuda")

    def run(ema, grouped):
        # tiny lr: every launch does the same work on almost the same values
        grp = {"groups": ug.chunk_groups, "group_hyper": ug.group_hyper} if grouped else {}
        co.adamw_split(hi, lo, m, v, grad, None, 1e-4, 0.9, 0.999, 1e-8, 0.1, 1, hyper,
                       ema=(ehi, elo) if ema else None, ema_decay=0.9998, **grp)

    variants = {f"{'ema_' if e else ''}{'grouped' if gr else 'plain'}": (lambda: None, (lambda e=e, gr=gr: run(e, gr)))
                for e in (False, True) for gr in (False, True)}
    times = time_alternating(variants, iters, warmup)
    rec = {"unit": f"ViT-10B {unit}", "W": W, "shard_numel": n, "groups": len(ug.rows), "grad": "float32"}
    for k, ts in times.items():
        ms = ts[len(ts) // 2]
        nbytes = adamw_bytes(n, 4, k.startswith("ema"), k.endswith("grouped"))
        rec[k] = {"ms_median": round(ms, 4), "ms_best": round(ts[0], 4), "bytes": nbytes,
                  "tb_per_s": round(nbytes / ms / 1e9, 3),
                  "share_of_3.35_datasheet": round(nbytes / ms / 1e9 / HBM_TBPS, 3)}
    rec["grouped_over_plain"] = round(rec["grouped"]["ms_median"] / rec["plain"]["ms_median"], 4)
    rec["ema_grouped_over_ema_plain"] = round(rec["ema_grouped"]["ms_median"] / rec["ema_plain"]["ms_median"], 4)
    print(json.dumps(rec), flush=True)
    del hi, lo, ehi, elo, m, v, grad
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_param_groups.py measures on the GPU; no CUDA device found")
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co

    info_before = gpu_info()
    print(json.dumps({"gpu_before": info_before}), flush=True)
    res = {"adamw_split": [bench_unit(co, unit, W, args.iters, args.warmup) for unit in ("block", "root")
                           for W in (4, 8)]}
    res["gpu_before"], res["gpu_after"] = info_before, gpu_info()
    print(json.dumps({"gpu_after": res["gpu_after"]}), flush=True)
    if args.out:
        if os.path.dirname(args.out):
            os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
