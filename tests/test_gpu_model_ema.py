"""Model EMA on the H100: the EMA operand of the AdamW kernels, the bf16 engine over three steps, CUDA graphs, the
EMA evaluation through the sm100 gathers (two or more GPUs) and a CLI run.

Bound of the device recurrence ema' = fmaf(d, ema, k * w), k = 1 - d in fp32: the stored EMA is exact fp32 (the split
into ema_hi / ema_lo is lossless), k * w is rounded once (u |k w|) and the fma once (u |ema'|), u = 2^-24.  A step's
error is carried into later steps multiplied by d < 1, so after T steps |ema - ema64| <= sum_t u (|k w_t| + |ema_t|),
with ema64 the fp64 recurrence with the same fp32 d and k over the masters w_t the kernel produced (recorded after every
step).  The checks below use twice that sum.  The inputs are normal numbers well away from the flush-to-zero range of
--use_fast_math."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def ema64_and_bound(init, masters, decay):
    d, k = float(np.float32(decay)), float(np.float32(1.0) - np.float32(decay))
    e = init.double().cpu().clone()
    bound = torch.zeros_like(e)
    for w in masters:
        w = w.double().cpu()
        e = d * e + k * w
        bound += 2 * U * ((k * w).abs() + e.abs())
    return e, bound


def _merge(hi, lo):
    out = torch.empty(hi.numel(), dtype=torch.float32, device=hi.device)
    _co().merge_fp32(hi, lo, out)
    return out


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a,
                       b.view(torch.int16) if b.dtype == torch.bfloat16 else b)


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4096, 4097, 4098, 4099, (1 << 20) + 3])
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("use_hyper", [False, True])
@pytest.mark.parametrize("decay", [0.9998, 0.9, 0.0])
def test_adamw_split_ema(n, gdt, use_hyper, decay):
    co = _co()
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(n)
    w0 = torch.randn(n, device=dev, generator=g) * 0.05
    hi, lo = torch.empty(n, dtype=torch.bfloat16, device=dev), torch.empty(n, dtype=torch.int16, device=dev)
    co.split_fp32(w0, hi, lo)
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    ref = [t.clone() for t in (hi, lo, m, v)]
    ehi, elo = hi.clone(), lo.clone()
    init = _merge(ehi, elo)
    clip = torch.tensor([0.7], device=dev)
    masters = []
    for step in range(1, 6):
        grad = (torch.randn(n, device=dev, generator=g) * 1e-2).to(gdt)
        hyper = torch.tensor([3e-3, float(step)], device=dev) if use_hyper else None
        lr = 10.0 if use_hyper else 3e-3  # with the device block the host lr / step must be ignored
        st = step + 7 if use_hyper else step
        co.adamw_split(hi, lo, m, v, grad, clip, lr, 0.9, 0.999, 1e-8, 0.1, st, hyper, ema=(ehi, elo), ema_decay=decay)
        co.adamw_split(*ref, grad, clip, lr, 0.9, 0.999, 1e-8, 0.1, st, hyper)
        masters.append(_merge(hi, lo))
    for a, b in zip((hi, lo, m, v), ref):  # the EMA operand changes nothing else
        assert _bits_equal(a, b)
    ema = _merge(ehi, elo)
    if decay == 0.0:
        assert torch.equal(ema, masters[-1])
        return
    e64, bound = ema64_and_bound(init, masters, decay)
    err = (ema.double().cpu() - e64).abs()
    assert bool((err <= bound).all()), f"worst {float((err - bound).max()):.3g}"


@pytest.mark.parametrize("n", [4097, 65536])
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("decay", [0.99, 0.0])
def test_adamw_fp32_ema(n, gdt, decay):
    co = _co()
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(n + 1)
    w = torch.randn(n, device=dev, generator=g) * 0.05
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    wr, mr, vr = w.clone(), m.clone(), v.clone()
    ema = w.clone()
    init = w.clone()
    masters = []
    for step in range(1, 6):
        grad = (torch.randn(n, device=dev, generator=g) * 1e-2).to(gdt)
        co.adamw_fp32(w, m, v, grad, None, 3e-3, 0.9, 0.999, 1e-8, 0.1, step, ema=ema, ema_decay=decay)
        co.adamw_fp32(wr, mr, vr, grad, None, 3e-3, 0.9, 0.999, 1e-8, 0.1, step)
        masters.append(w.clone())
    assert torch.equal(w, wr) and torch.equal(m, mr) and torch.equal(v, vr)
    if decay == 0.0:
        assert torch.equal(ema, w)
        return
    e64, bound = ema64_and_bound(init, masters, decay)
    assert bool(((ema.double().cpu() - e64).abs() <= bound).all())


def test_rejects_bad_ema_arguments():
    co = _co()
    dev = torch.device("cuda")
    n = 64
    hi, lo = torch.zeros(n, dtype=torch.bfloat16, device=dev), torch.zeros(n, dtype=torch.int16, device=dev)
    m, v, grad = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    with pytest.raises(RuntimeError, match="as many elements"):
        co.adamw_split(hi, lo, m, v, grad, None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1, ema=(hi[:32], lo[:32]), ema_decay=0.9)
    with pytest.raises(RuntimeError, match="ema_hi must be bf16"):
        co.adamw_split(hi, lo, m, v, grad, None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1, ema=(lo, hi), ema_decay=0.9)
    with pytest.raises(RuntimeError, match=r"ema_decay must be in \[0, 1\)"):
        co.adamw_split(hi, lo, m, v, grad, None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1, ema=(hi.clone(), lo.clone()),
                       ema_decay=1.0)
    with pytest.raises(RuntimeError, match="contiguous fp32"):
        co.adamw_fp32(m, v, grad.clone(), grad, None, 1e-3, 0.9, 0.999, 1e-8, 0.1, 1, ema=hi, ema_decay=0.9)


# ------------------------------------------------------------------------------------------------
# the bf16 engine on one GPU
# ------------------------------------------------------------------------------------------------
def _cfg():
    from vit_10b_fsdp_example_b200.config import ViTConfig

    return ViTConfig(image_size=112, patch_size=14, embed_dim=320, num_heads=2, num_blocks=2, mlp_ratio=4.0,
                     num_classes=96)


def _data(n=3, B=8):
    g = torch.Generator().manual_seed(0)
    return [(torch.randn(B, 3, 112, 112, generator=g).cuda(), torch.randint(0, 96, (B,), generator=g).cuda())
            for _ in range(n)]


def _model(ema, decay=0.99):
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW

    model = FSDPViT(_cfg(), device=torch.device("cuda"), dtype=torch.bfloat16, seed=4, model_ema=ema)
    opt = ShardedAdamW(model, lr=2e-3, weight_decay=0.1, model_ema_decay=decay if ema else None)
    return model, opt


def _consolidated(model, sd):
    from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate

    return consolidate([{"shard_metadata": model.get_shard_metadata(), "model": sd}])


def test_three_steps_match_the_run_without_the_flag_and_the_host_recurrence():
    """Same seed, same data, with and without the flag: the forward / backward kernels are the same with or without
    the EMA, so any difference would come from the GEMMs' atomics; what is compared bitwise is the optimizer's output
    from identical inputs, step by step (both models are reset to the same master and moments before each step)."""
    data = _data()
    on, opt_on = _model(True)
    off, opt_off = _model(False)
    init = [on.master_fp32(u).clone() for u in on.all_units]
    masters = [[] for _ in on.all_units]
    for x, y in data:
        loss_on = on.forward_backward(x, y)
        # the same gradients in both models: the comparison is of the update, not of GEMM atomics order
        for a, b in zip(on.all_units, off.all_units):
            b.shard_grad.copy_(a.shard_grad)
            b.hi.copy_(a.hi), b.lo.copy_(a.lo), b.exp_avg.copy_(a.exp_avg), b.exp_avg_sq.copy_(a.exp_avg_sq)
        off.step_count = on.step_count
        on.clip_grad_norm_(1.0)
        off._clip_coef = on._clip_coef.clone()
        opt_on.step()
        opt_off.step()
        assert torch.isfinite(loss_on)
        for i, (a, b) in enumerate(zip(on.all_units, off.all_units)):
            for t in ("hi", "lo", "exp_avg", "exp_avg_sq"):
                assert _bits_equal(getattr(a, t), getattr(b, t)), (a.name, t)
            masters[i].append(on.master_fp32(a).clone())
    for i, u in enumerate(on.all_units):
        e64, bound = ema64_and_bound(init[i], masters[i], 0.99)
        err = (on.ema_fp32(u).double().cpu() - e64).abs()
        assert bool((err <= bound).all()), (u.name, float((err - bound).max()))


def test_training_loss_is_unchanged_by_the_flag():
    """Whole steps with and without the flag, from the same seed and data.

    The forward before any update is bitwise the same (its logits are compared).  The scalar loss is not: the
    cross-entropy kernel adds the B per-row terms t_b = (lse_b - logit_b[y_b]) / B to one float with atomicAdd, in the
    order the rows finish, so two runs of the same model may differ in its last bits.  Each t_b is computed the same way
    in both runs (one CTA per row) and t_b >= 0, so two summation orders of the B terms differ by at most
    2 (B - 1) u sum_b t_b = 2 (B - 1) u loss (u = 2^-24, each of the B - 1 fp32 additions rounds once, relative to a
    partial sum <= loss).  Later steps start from updates whose gradients carry the GEMMs' atomics-order noise as well;
    they are held to the tolerance the engine's graphed-against-eager test uses for trajectories that differ only in
    that order.  That the update itself is bitwise unchanged by the EMA is checked above from identical inputs."""
    data = _data()
    runs = []
    for ema in (True, False):
        model, opt = _model(ema)
        logits = model.eval()(data[0][0])
        model.train()
        losses = []
        for x, y in data:
            losses.append(model.forward_backward(x, y).item())
            model.clip_grad_norm_(1.0)
            opt.step()
        runs.append((logits, losses))
    (lg_on, on), (lg_off, off) = runs
    assert torch.equal(lg_on, lg_off)
    B = data[0][0].shape[0]
    assert abs(on[0] - off[0]) <= 2 * (B - 1) * U * abs(off[0]), (on[0], off[0])
    for a, b in zip(on, off):
        assert abs(a - b) < 2e-2 * abs(b) + 1e-3, (on, off)


def test_ema_evaluation_equals_a_model_loaded_with_the_ema():
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    model, opt = _model(True)
    for x, y in _data():
        model.forward_backward(x, y)
        model.clip_grad_norm_(1.0)
        opt.step()
    images = _data(1, B=6)[0][0]
    model.eval()
    before = model(images)
    with model.ema_weights():
        got = model(images)
    after = model(images)
    loaded = FSDPViT(_cfg(), device=torch.device("cuda"), dtype=torch.bfloat16, seed=9)
    loaded.load_full_state_dict(_consolidated(model, model.ema_state_dict()))
    want = loaded.eval()(images)
    assert torch.equal(got, want)
    assert torch.equal(before, after) and not torch.equal(got, before)


def test_cuda_graph_updates_the_ema_like_eager_steps():
    """The optimizer step replayed from a CUDA graph (device lr / step, the EMA operand recorded once) gives bitwise the
    EMA of eager steps from the same gradients; and a whole graphed training step composes with the EMA."""
    from vit_10b_fsdp_example_b200.parallel import GraphedTrainStep

    data = _data()
    a, opt_a = _model(True)
    b, opt_b = _model(True)
    a.forward_backward(*data[0])
    for ua, ub in zip(a.all_units, b.all_units):
        ub.shard_grad.copy_(ua.shard_grad)
    lrs = [2e-3, 1.5e-3, 1e-3, 5e-4]
    for lr in lrs:  # eager
        opt_a.param_groups[0]["lr"] = lr
        opt_a.step()
    opt_b.lr_on_device = True
    opt_b.param_groups[0]["lr"] = lrs[0]
    opt_b.push_lr()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt_b.step()
    for lr in lrs:
        opt_b.param_groups[0]["lr"] = lr
        opt_b.push_lr()
        graph.replay()
    torch.cuda.synchronize()
    for ua, ub in zip(a.all_units, b.all_units):
        for t in ("hi", "lo", "ema_hi", "ema_lo", "exp_avg", "exp_avg_sq"):
            assert _bits_equal(getattr(ua, t), getattr(ub, t)), (ua.name, t)
    # a whole graphed step: the EMA follows the recurrence over the masters the graph produced
    model, opt = _model(True)
    step = GraphedTrainStep(model, opt, clip_grad_norm=1.0, warmup=2)
    init = [model.master_fp32(u).clone() for u in model.all_units]
    masters = [[] for _ in model.all_units]
    for i in range(5):
        step(*data[i % 3])
        for j, u in enumerate(model.all_units):
            masters[j].append(model.master_fp32(u).clone())
    assert step.graph is not None
    for j, u in enumerate(model.all_units):
        e64, bound = ema64_and_bound(init[j], masters[j], 0.99)
        assert bool(((model.ema_fp32(u).double().cpu() - e64).abs() <= bound).all()), u.name


# ------------------------------------------------------------------------------------------------
# two or more GPUs: the EMA evaluation through the symmetric ema_hi and the AG-fused GEMMs
# ------------------------------------------------------------------------------------------------
def _multi_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    dev = torch.device("cuda", rank)
    model = FSDPViT(_cfg(), world=world, rank=rank, device=dev, dtype=torch.bfloat16, backend="sm100", seed=4,
                    model_ema=True)
    opt = ShardedAdamW(model, lr=2e-3, weight_decay=0.1, model_ema_decay=0.9)
    for x, y in _data():
        model.forward_backward(x.to(dev)[rank::world], y.to(dev)[rank::world])
        model.clip_grad_norm_(1.0)
        opt.step()
    images = _data(1, B=6)[0][0].to(dev)
    model.eval()
    before = model(images)
    with model.ema_weights():
        got = model(images)
    after = model(images)
    torch.save({"model": model.ema_state_dict(), "shard_metadata": model.get_shard_metadata(), "logits": got.cpu(),
                "same_after": bool(torch.equal(before, after)), "fused": bool(model.fuse_all_gather)},
               os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_sm100_ema_evaluation_matches_one_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    from helpers import free_port
    from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    mp.spawn(_multi_worker, args=(2, free_port(), str(tmp_path)), nprocs=2, join=True)
    recs = [torch.load(str(tmp_path / f"r{r}.pt"), weights_only=False) for r in range(2)]
    assert all(r["same_after"] for r in recs)
    ema = consolidate(recs)
    one = FSDPViT(_cfg(), device=torch.device("cuda"), dtype=torch.bfloat16, seed=0)
    one.load_full_state_dict(ema)
    want = one.eval()(_data(1, B=6)[0][0]).float().cpu()
    for r in recs:
        got = r["logits"].float()
        # the same bf16 weights and kernels; only the GEMMs' fp32 accumulation order may differ: one bf16 ulp of the
        # largest logit
        assert (got - want).abs().max().item() <= 2.0 ** -7 * want.abs().max().item(), (got - want).abs().max()


# ------------------------------------------------------------------------------------------------
# CLI
# ------------------------------------------------------------------------------------------------
def test_cli_trains_evaluates_checkpoints_and_resumes_with_the_ema(tmp_path):
    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "16",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--model_ema", "--model_ema_decay", "0.9",
            "--ckpt_dir", str(tmp_path)]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")

    def run(*extra):
        r = subprocess.run([sys.executable, "run_vit_training.py", *args, *extra], cwd=ROOT, env=env,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        return r.stdout

    out = run("--num_epochs", "2")
    assert out.count("accuracy on val: ") == 2 and out.count("accuracy of the EMA on val: ") == 2
    ck = torch.load(str(tmp_path / "epoch_1_rank_0.ckpt"), weights_only=False)
    assert set(ck) == {"model", "shard_metadata", "optimizer", "lr_scheduler", "model_ema"}
    assert ck["model_ema"].keys() == ck["model"].keys()
    assert any(not torch.equal(ck["model_ema"][k], ck["model"][k]) for k in ck["model"])
    out = run("--num_epochs", "3", "--resume_epoch", "2")
    assert "resumed from checkpoint" in out and "no model_ema" not in out
    assert out.count("accuracy of the EMA on val: ") == 1
    assert "model_ema" in torch.load(str(tmp_path / "epoch_3_rank_0.ckpt"), weights_only=False)
