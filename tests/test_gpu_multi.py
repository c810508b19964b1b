"""Multi-GPU tests of the NVLink symmetric-memory collectives and the sm100 FSDP backend.

Needs >= 2 GPUs (skipped otherwise): `python -m pytest tests/test_gpu_multi.py -m gpu`.
Custom all-gather must be bit-exact vs NCCL; reduce-scatter within fp32 reorder tolerance; flags are reused
for >= 1000 iterations to catch phase bugs.
"""
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _need_gpus(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} GPUs")


def _init(rank, world, port):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    return dist


def _collectives_worker(rank, world, port, out_path):
    dist = _init(rank, world, port)
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.models import vit
    from vit_10b_fsdp_example_b200.ops import cuda_ops
    from vit_10b_fsdp_example_b200.parallel.backends import Sm100Backend, TorchDistBackend
    from vit_10b_fsdp_example_b200.parallel.layout import UnitLayout

    dev = torch.device("cuda", rank)
    sm = Sm100Backend(world, rank, dev)
    nc = TorchDistBackend(world, rank, dev)
    res = {"nvls": bool(sm.use_nvls)}
    cfg = ViTConfig(embed_dim=640, num_heads=4, num_blocks=1)
    for flatten in (False, True):
        lay = UnitLayout.build("blocks.0", vit.block_param_specs(cfg), world, flatten)
        torch.manual_seed(100 + rank)
        shard = sm.alloc_shard(lay.shard_numel, torch.bfloat16)
        shard.copy_(torch.randn(lay.shard_numel, device=dev))
        sm.params_updated()
        full_a = torch.zeros(lay.full_numel, dtype=torch.bfloat16, device=dev)
        full_b = torch.zeros(lay.full_numel, dtype=torch.bfloat16, device=dev)
        nc.all_gather(lay, shard, full_b)
        ok_ag = True
        for transport in ("kernel", "ce"):  # light pull kernel and copy-engine transport of the all-gather
            sm.ag_transport = transport
            full_a.zero_()
            sm.all_gather(lay, shard, full_a)
            torch.cuda.synchronize()
            ok_ag = ok_ag and bool(torch.equal(full_a, full_b))
        res[f"ag_exact_{int(flatten)}"] = ok_ag
        # reduce-scatter: P2P and (if available) NVLS vs NCCL fp32
        grad = sm.alloc_full_grad(lay.full_numel, torch.bfloat16)
        grad.copy_(torch.randn(lay.full_numel, device=dev))
        torch.cuda.synchronize()
        dist.barrier()
        ref = torch.zeros(lay.shard_numel, dtype=torch.float32, device=dev)
        ssq_ref = torch.zeros(1, device=dev)
        nc.reduce_scatter(lay, grad, ref, ssq_ref, cuda_ops)
        for mode in ("p2p", "nvls"):
            if mode == "nvls" and not sm.use_nvls:
                continue
            saved = sm.use_nvls
            sm.use_nvls = mode == "nvls"
            out = torch.zeros(lay.shard_numel, dtype=torch.float32, device=dev)
            ssq = torch.zeros(1, device=dev)
            sm.reduce_scatter(lay, grad, out, ssq, cuda_ops)
            torch.cuda.synchronize()
            sm.use_nvls = saved
            tol = 1e-6 if mode == "p2p" else 2e-2  # NVLS returns the fp32 sum rounded to bf16
            err = (out - ref).abs().max().item()
            res[f"rs_{mode}_err_{int(flatten)}"] = err
            res[f"rs_{mode}_ok_{int(flatten)}"] = bool(err <= tol * (ref.abs().max().item() + 1e-6) + 1e-7)
            res[f"rs_{mode}_ssq_ok_{int(flatten)}"] = bool(abs(ssq.item() - ssq_ref.item()) <= 2e-2 * ssq_ref.item())
    # in-kernel flag protocol of the reduce-scatter reused for > 1000 back-to-back calls on two alternating buffers
    # (sequence-number / last-CTA-counter / phase bugs), checked against the fp32 reference every 100 calls
    lay = UnitLayout.build("blocks.0", vit.block_param_specs(cfg), world, False)
    bufs = [sm.alloc_full_grad(lay.full_numel, torch.bfloat16) for _ in range(2)]
    out = torch.zeros(lay.shard_numel, dtype=torch.float32, device=dev)
    ok_loop = True
    for it in range(1050):
        g = bufs[it & 1]
        if it % 100 == 0:
            g.copy_(torch.randn(lay.full_numel, device=dev) * (1.0 + it / 100.0))
        sm.reduce_scatter(lay, g, out, None, cuda_ops)
        if it % 100 == 0:
            ref = torch.zeros(lay.shard_numel, dtype=torch.float32, device=dev)
            nc.reduce_scatter(lay, g, ref, None, cuda_ops)
            torch.cuda.synchronize()
            err = (out - ref).abs().max().item()
            ok_loop = ok_loop and err <= 2e-2 * (ref.abs().max().item() + 1e-6)
    res["rs_flag_reuse_ok"] = bool(ok_loop)
    # DDP gradient all-reduce (mean) on the symmetric buffer: in-switch (NVLS) and pull-reduce-push variants vs NCCL
    for mode in ("p2p", "nvls"):
        if mode == "nvls" and not sm.use_nvls:
            continue
        saved = sm.use_nvls
        sm.use_nvls = mode == "nvls"
        g = bufs[0]
        torch.manual_seed(500 + rank)
        g.copy_(torch.randn(lay.full_numel, device=dev))
        ref = g.float()
        torch.cuda.synchronize()
        dist.barrier()
        dist.all_reduce(ref)
        ref.mul_(1.0 / world)
        sm.all_reduce_mean_(g)
        torch.cuda.synchronize()
        sm.use_nvls = saved
        err = (g.float() - ref).abs().max().item()
        res[f"ar_{mode}_err"] = err
        res[f"ar_{mode}_ok_0"] = bool(err <= 1.6e-2 * (ref.abs().max().item() + 1e-6))
        # every rank must hold bit-identical results (replicated parameters stay replicated)
        chk = g.view(torch.int16).to(torch.int64).sum().reshape(1)
        lo, hi = chk.clone(), chk.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        res[f"ar_{mode}_identical_ok_0"] = bool(lo.item() == hi.item())
    dist.barrier()
    # all-gather fused into the consuming GEMM: y = x @ W^T where W's row slabs live on the peers
    Nw, Kw, Mx = 2048, 512, 1024
    torch.manual_seed(7)
    w_full = (torch.randn(Nw, Kw, device=dev) * 0.05).to(torch.bfloat16)   # identical on every rank (same seed)
    rows = Nw // world
    w_shard = sm.alloc_shard(rows * Kw, torch.bfloat16)
    w_shard.copy_(w_full[rank * rows:(rank + 1) * rows].reshape(-1))
    sm.params_updated()
    torch.cuda.synchronize()
    dist.barrier()
    xin = torch.randn(Mx, Kw, device=dev).to(torch.bfloat16)
    bias = torch.randn(Nw, device=dev).to(torch.bfloat16)
    ref = cuda_ops.linear_fwd(xin, w_full, bias)
    flags = torch.zeros(16, dtype=torch.int32, device=dev)
    ok_fused = True
    for it in range(5):
        gathered = torch.zeros(Nw, Kw, dtype=torch.bfloat16, device=dev)
        spec = [world, rank, rows, rows * Kw * 2, gathered.data_ptr(), flags.data_ptr()] + list(sm._peer[w_shard.data_ptr()])
        y = cuda_ops.linear_fwd(xin, gathered, bias, ag=spec)
        torch.cuda.synchronize()
        ok_fused = ok_fused and bool(torch.equal(gathered, w_full)) and bool(torch.equal(y, ref))
    res["ag_fused_gemm_exact"] = ok_fused
    dist.barrier()
    # scalar all-reduce + barrier reuse for > 1000 iterations (sequence-number / phase bugs)
    ok = True
    for it in range(1100):
        v = torch.tensor([float(rank + it), 1.0], device=dev)
        sm.all_reduce_scalars_(v, "sum")
        if it % 97 == 0:
            sm.device_barrier(0)
        if it % 100 == 0 or it == 1099:
            exp = sum(r + it for r in range(world))
            ok = ok and abs(v[0].item() - exp) < 1e-3 and abs(v[1].item() - world) < 1e-6
    m = torch.tensor([float(rank)], device=dev)
    sm.all_reduce_scalars_(m, "max")
    res["scalars_ok"] = bool(ok and m.item() == world - 1)
    torch.cuda.synchronize()
    dist.barrier()
    if rank == 0:
        json.dump(res, open(out_path, "w"))
    dist.destroy_process_group()


def _train_worker(rank, world, port, backend, out_path, flatten, reshard, clip=1.0, fuse_opt=False, graph=False,
                  ddp=False):
    dist = _init(rank, world, port)
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW

    dev = torch.device("cuda", rank)
    cfg = ViTConfig(image_size=112, patch_size=14, embed_dim=320, num_heads=2, num_blocks=3, mlp_ratio=4.0,
                    num_classes=96)
    model = FSDPViT(cfg, world=world, rank=rank, device=dev, dtype=torch.bfloat16, backend=backend, seed=1,
                    flatten_parameters=flatten, reshard_after_forward=reshard, run_without_fsdp=ddp)
    opt = ShardedAdamW(model, lr=1e-3, weight_decay=0.1, fuse_into_reduce_scatter=fuse_opt)
    assert opt.fused == (fuse_opt and backend == "sm100")
    g = torch.Generator().manual_seed(0)
    images = torch.randn(16, 3, 112, 112, generator=g)
    target = torch.randint(0, 96, (16,), generator=g)
    lb = 16 // world
    losses, norms = [], []
    gstep = None
    if graph:
        from vit_10b_fsdp_example_b200.parallel import GraphedTrainStep

        gstep = GraphedTrainStep(model, opt, clip_grad_norm=clip, warmup=2)
    for _ in range(6):
        xi, yi = images[rank * lb:(rank + 1) * lb].to(dev), target[rank * lb:(rank + 1) * lb].to(dev)
        if gstep is not None:
            loss = gstep(xi, yi)
            norm = gstep.grad_norm if gstep.grad_norm is not None else torch.zeros(1)
        else:
            loss = model.forward_backward(xi, yi)
            norm = model.clip_grad_norm_(clip) if clip > 0 else torch.zeros(1)
            opt.step()
        lv = loss.detach().float().reshape(1).clone()
        dist.all_reduce(lv)
        losses.append(lv.item() / world)
        norms.append(norm.item())
    # inference right after the last optimizer step, with NO host synchronisation in between: the eval gathers must
    # be ordered after AdamW and its cross-GPU barrier (ADVICE r1); compare with the same pass after a full sync
    model.eval()
    logits_a = model(xi).float().clone()
    torch.cuda.synchronize()
    dist.barrier()
    logits_b = model(xi).float()
    eval_err = (logits_a - logits_b).abs().max().item()
    model.train()
    torch.cuda.synchronize()
    dist.barrier()
    if rank == 0:
        json.dump({"losses": losses, "norms": norms, "eval_err": eval_err}, open(out_path, "w"))
    dist.destroy_process_group()


def _spawn(fn, world, args):
    import torch.multiprocessing as mp
    from helpers import free_port

    mp.spawn(fn, args=(world, free_port()) + args, nprocs=world, join=True)


def _worlds():
    """World sizes to test: 2 always (skipped without 2 GPUs), plus 4 / 8 when the box has them."""
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    return [w for w in (2, 4, 8) if w <= max(n, 2)]


def _train_world():
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    return 8 if n >= 8 else (4 if n >= 4 else 2)


@pytest.mark.parametrize("world", _worlds())
def test_symmetric_memory_collectives(world, tmp_path):
    _need_gpus(world)
    out = str(tmp_path / "c.json")
    _spawn(_collectives_worker, world, (out,))
    res = json.load(open(out))
    print(res)
    bad = [k for k, v in res.items()
           if k.endswith(("_ok_0", "_ok_1", "exact_0", "exact_1", "scalars_ok", "ag_fused_gemm_exact",
                          "rs_flag_reuse_ok")) and not v]
    assert not bad, (bad, res)


@pytest.mark.parametrize("flatten,reshard", [(False, True), (True, False)])
def test_sm100_backend_matches_nccl_backend(flatten, reshard, tmp_path):
    world = _train_world()
    _need_gpus(world)
    outs = {}
    for backend in ("torchdist", "sm100"):
        out = str(tmp_path / f"{backend}.json")
        _spawn(_train_worker, world, (backend, out, flatten, reshard))
        outs[backend] = json.load(open(out))
    a, b = outs["torchdist"], outs["sm100"]
    for x, y in zip(a["losses"], b["losses"]):
        assert abs(x - y) < 0.03 * abs(x) + 0.02, (a, b)
    for x, y in zip(a["norms"], b["norms"]):
        assert abs(x - y) < 0.05 * abs(x) + 0.02, (a, b)
    assert b["losses"][-1] < b["losses"][0]
    assert min(b["norms"]) > 1e-3, "gradients must be non-degenerate for this comparison to mean anything"
    assert b["eval_err"] == 0.0, f"eval right after the optimizer step read stale / in-flight shards: {b['eval_err']}"


def test_ddp_all_reduce_on_symmetric_memory(tmp_path):
    """--run_without_fsdp: replicated parameters, gradient all-reduce on the hand-written NVLS / P2P kernel vs NCCL."""
    world = 2
    _need_gpus(world)
    outs = {}
    for backend in ("torchdist", "sm100"):
        out = str(tmp_path / f"{backend}.json")
        _spawn(_train_worker, world, (backend, out, False, True, 1.0, False, False, True))
        outs[backend] = json.load(open(out))
    a, b = outs["torchdist"], outs["sm100"]
    for x, y in zip(a["losses"], b["losses"]):
        assert abs(x - y) < 0.03 * abs(x) + 0.02, (a, b)
    for x, y in zip(a["norms"], b["norms"]):
        assert abs(x - y) < 0.05 * abs(x) + 0.02, (a, b)
    assert b["losses"][-1] < b["losses"][0]


def test_adamw_fused_into_reduce_scatter(tmp_path):
    """Clipping off: the AdamW update runs inside each unit's reduce-scatter kernel during backward and must give
    the same trajectory as the separate optimizer step on the NCCL backend."""
    world = 2
    _need_gpus(world)
    outs = {}
    for name, backend, fuse in (("ref", "torchdist", False), ("fused", "sm100", True)):
        out = str(tmp_path / f"{name}.json")
        _spawn(_train_worker, world, (backend, out, False, True, 0.0, fuse))
        outs[name] = json.load(open(out))
    a, b = outs["ref"], outs["fused"]
    for x, y in zip(a["losses"], b["losses"]):
        assert abs(x - y) < 0.03 * abs(x) + 0.02, (a, b)
    assert b["losses"][-1] < b["losses"][0]


def test_cuda_graph_step_two_gpus(tmp_path):
    """Whole step (incl. the symmetric-memory collectives with device-side sequence numbers) as one CUDA graph."""
    world = 2
    _need_gpus(world)
    outs = {}
    for name, graph in (("eager", False), ("graph", True)):
        out = str(tmp_path / f"{name}.json")
        _spawn(_train_worker, world, ("sm100", out, False, True, 1.0, False, graph))
        outs[name] = json.load(open(out))
    a, b = outs["eager"], outs["graph"]
    for x, y in zip(a["losses"], b["losses"]):
        assert abs(x - y) < 0.03 * abs(x) + 0.02, (a, b)
    assert b["losses"][-1] < b["losses"][0]
    # eager inference after graph replays (events recorded during capture must not leak into eager waits)
    assert b["eval_err"] == 0.0, b
