"""Model EMA (--model_ema / --model_ema_decay): timm ModelEmaV2 with a fixed decay, sharded like the master and updated
by the AdamW step.  CPU checks: the flags, the torch_ops recurrence against fp64, training on fp32 CPU at W = 1 and on
gloo at W = 2 (flattened and not), checkpoints, consolidation, --init_from_full_ckpt and the evaluation swap.

Error bound of the fp32 recurrence ema' = fmaf(d, ema, k * w), k = 1 - d (d and k fp32, k exact by Sterbenz for
d >= 0.5): the product k * w is rounded once (u |k w|) and the fused add once (u |ema'|), u = 2^-24.  torch_ops emulates
the fma in fp64 and rounds the fp64 sum to fp32, which adds at most one more u |ema'|.  A per-step error is carried into
later steps multiplied by d < 1, so after T steps |ema - ema64| <= sum_t u (|k w_t| + 2 |ema_t|) elementwise, with ema64
the fp64 recurrence with the same fp32 d and k over the same recorded masters w_t."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import free_port, tiny_cfg
from vit_10b_fsdp_example_b200.config import parse_args
from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate, consolidate_files
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW
from vit_10b_fsdp_example_b200.utils import get_warmup_cosine_scheduler
from vit_10b_fsdp_example_b200.utils.checkpoint import load_ckpt, save_ckpt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
STEPS = 5


def fp32_pair(d):
    """(d, 1 - d) as the device forms them: d rounded to fp32, 1 - d subtracted in fp32."""
    return float(np.float32(d)), float(np.float32(1.0) - np.float32(d))


def ema64_and_bound(init, masters, decay):
    """fp64 recurrence over the recorded fp32 masters and the elementwise bound of the module docstring."""
    d, k = fp32_pair(decay)
    e = init.double().clone()
    bound = torch.zeros_like(e)
    for w in masters:
        e = d * e + k * w.double()
        bound += U * ((k * w.double()).abs() + 2 * e.abs())
    return e, bound


# ------------------------------------------------------------------------------------------------
# flags
# ------------------------------------------------------------------------------------------------
def test_flag_defaults_and_validation():
    a = parse_args([])
    assert a.model_ema is False and a.model_ema_decay == 0.9998
    a = parse_args(["--model_ema", "--model_ema_decay", "0.99996"])
    assert a.model_ema is True and a.model_ema_decay == 0.99996
    assert parse_args(["--model_ema_decay", "0"]).model_ema_decay == 0.0
    for bad in ("1", "1.5", "-0.1", "nan", "inf"):
        with pytest.raises(SystemExit):
            parse_args(["--model_ema_decay", bad])


def test_optimizer_refuses_a_decay_that_does_not_match_the_model():
    with_ema = FSDPViT(tiny_cfg(), dtype=torch.float32, model_ema=True)
    without = FSDPViT(tiny_cfg(), dtype=torch.float32)
    with pytest.raises(ValueError, match="has an EMA: pass model_ema_decay"):
        ShardedAdamW(with_ema)
    with pytest.raises(ValueError, match="needs a model with an EMA"):
        ShardedAdamW(without, model_ema_decay=0.9)
    with pytest.raises(ValueError, match=r"must be in \[0, 1\)"):
        ShardedAdamW(with_ema, model_ema_decay=1.0)
    with pytest.raises(RuntimeError, match="has no EMA"):
        with without.ema_weights():
            pass


# ------------------------------------------------------------------------------------------------
# torch_ops: the recurrence against fp64
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("decay", [0.9998, 0.99996, 0.9, 0.5])
def test_torch_ops_adamw_ema_against_fp64(decay):
    g = torch.Generator().manual_seed(3)
    n = 4099
    w = torch.randn(n, generator=g) * torch.logspace(-3, 1, n)
    m, v = torch.zeros(n), torch.zeros(n)
    ema = w.clone()
    init = w.clone()
    w_ref, m_ref, v_ref = w.clone(), m.clone(), v.clone()
    masters = []
    for step in range(1, 61):
        grad = torch.randn(n, generator=g)
        torch_ops.adamw_fp32(w, m, v, grad, None, 1e-2, 0.9, 0.999, 1e-8, 0.1, step, ema=ema, ema_decay=decay)
        torch_ops.adamw_fp32(w_ref, m_ref, v_ref, grad, None, 1e-2, 0.9, 0.999, 1e-8, 0.1, step)
        masters.append(w.clone())
    assert torch.equal(w, w_ref) and torch.equal(m, m_ref) and torch.equal(v, v_ref)  # the EMA changes nothing else
    e64, bound = ema64_and_bound(init, masters, decay)
    err = (ema.double() - e64).abs()
    assert bool((err <= bound).all()), float((err - bound).max())
    assert float(err.max()) > 0 or decay == 0.5  # the check is not vacuous: fp32 really rounds


def test_torch_ops_adamw_split_ema():
    """Split form: hi / lo / m / v are bitwise those of the plain update; the EMA follows the fp32 recurrence on the
    merged value; d = 0 copies the master bitwise."""
    g = torch.Generator().manual_seed(4)
    n = 1027
    w0 = torch.randn(n, generator=g)
    for decay in (0.999, 0.0):
        hi, lo = torch.empty(n, dtype=torch.bfloat16), torch.empty(n, dtype=torch.int16)
        torch_ops.split_fp32(w0, hi, lo)
        ehi, elo = hi.clone(), lo.clone()
        hr, lr_, m, v, mr, vr = hi.clone(), lo.clone(), torch.zeros(n), torch.zeros(n), torch.zeros(n), torch.zeros(n)
        e = w0.clone()
        for step in range(1, 4):
            grad = torch.randn(n, generator=g)
            torch_ops.adamw_split(hi, lo, m, v, grad, None, 1e-2, 0.9, 0.999, 1e-8, 0.1, step, ema=(ehi, elo),
                                  ema_decay=decay)
            torch_ops.adamw_split(hr, lr_, mr, vr, grad, None, 1e-2, 0.9, 0.999, 1e-8, 0.1, step)
            w = torch.empty(n)
            torch_ops.merge_fp32(hi, lo, w)
            torch_ops.ema_update(e, w, decay)
        assert torch.equal(hi.view(torch.int16), hr.view(torch.int16)) and torch.equal(lo, lr_)
        assert torch.equal(m, mr) and torch.equal(v, vr)
        got = torch.empty(n)
        torch_ops.merge_fp32(ehi, elo, got)
        assert torch.equal(got, e)
        if decay == 0.0:
            assert torch.equal(got, w)


# ------------------------------------------------------------------------------------------------
# training on fp32 CPU: W = 1 and W = 2 on gloo, flattened and not
# ------------------------------------------------------------------------------------------------
def _train_worker(rank, world, port, opts, out):
    torch.set_num_threads(1)
    if world > 1:
        import torch.distributed as dist

        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg = tiny_cfg()
    ema = opts.get("decay") is not None
    model = FSDPViT(cfg, world=world, rank=rank, dtype=torch.float32, flatten_parameters=opts.get("flatten", False),
                    seed=1, model_ema=ema)
    opt = ShardedAdamW(model, lr=1e-2, weight_decay=0.1, model_ema_decay=opts.get("decay"))
    g = torch.Generator().manual_seed(1234)
    images = torch.randn(STEPS, 8, 3, cfg.image_size, cfg.image_size, generator=g)
    targets = torch.randint(0, cfg.num_classes, (STEPS, 8), generator=g)
    local = 8 // world
    rec = {"losses": [], "masters": [model.state_dict()], "md": model.get_shard_metadata()}
    for s in range(STEPS):
        loss = model.forward_backward(images[s, rank * local:(rank + 1) * local],
                                      targets[s, rank * local:(rank + 1) * local])
        model.clip_grad_norm_(1.0)
        opt.step()
        rec["losses"].append(loss.clone())
        rec["masters"].append(model.state_dict())
    rec["optimizer"] = opt.state_dict()
    if ema:
        rec["ema"] = model.ema_state_dict()
    torch.save(rec, out.format(rank=rank))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def _train(tmp, world, **opts):
    out = os.path.join(tmp, f"w{world}_{opts.get('flatten', False)}_{opts.get('decay')}_rank_{{rank}}.pt")
    if world == 1:
        _train_worker(0, 1, 0, opts, out)
    else:
        import torch.multiprocessing as mp

        mp.spawn(_train_worker, args=(world, free_port(), opts, out), nprocs=world, join=True)
    return [torch.load(out.format(rank=r), weights_only=False) for r in range(world)]


def _full(recs, key, i=None):
    """Consolidated (timm-layout) state of the ranks' recorded `key` (step i of the master history)."""
    return consolidate([{"shard_metadata": r["md"], "model": r[key] if i is None else r[key][i]} for r in recs])


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp("ema_runs"))
    out = {}
    for world in (1, 2):
        for flatten in (False, True):
            for decay in (None, 0.9):
                out[(world, flatten, decay)] = _train(tmp, world, flatten=flatten, decay=decay)
    out[(1, False, 0.0)] = _train(tmp, 1, decay=0.0)
    return out


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("flatten", [False, True])
def test_training_is_bitwise_unchanged_and_the_ema_follows_the_recurrence(runs, world, flatten):
    on, off = runs[(world, flatten, 0.9)], runs[(world, flatten, None)]
    for a, b in zip(on, off):  # every rank: losses, master history, moments
        assert all(torch.equal(x, y) for x, y in zip(a["losses"], b["losses"]))
        for sa, sb in zip(a["masters"], b["masters"]):
            assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)
        for name, st in a["optimizer"]["state"].items():
            sb = b["optimizer"]["state"][name]
            assert st["step"] == sb["step"]
            assert torch.equal(st["exp_avg"], sb["exp_avg"]) and torch.equal(st["exp_avg_sq"], sb["exp_avg_sq"])
    ema = _full(on, "ema")
    init = _full(on, "masters", 0)
    masters = [_full(on, "masters", i) for i in range(1, STEPS + 1)]
    for k in ema:
        e64, bound = ema64_and_bound(init[k].reshape(-1), [m[k].reshape(-1) for m in masters], 0.9)
        err = (ema[k].reshape(-1).double() - e64).abs()
        assert bool((err <= bound).all()), (k, float((err - bound).max()))


def test_zero_decay_gives_the_master_bitwise(runs):
    (rec,) = runs[(1, False, 0.0)]
    last = rec["masters"][-1]
    assert all(torch.equal(rec["ema"][k], last[k]) for k in last)


@pytest.mark.parametrize("flatten", [False, True])
def test_consolidated_ema_does_not_depend_on_the_world_size(runs, flatten):
    """The W = 2 masters differ from W = 1 only by the order of the gradient reduction; the EMA is a convex combination
    of the masters (weights d^T, (1 - d) d^(T - t)), so its difference is bounded by the largest master difference over
    the steps plus both rounding bounds."""
    r1, r2 = runs[(1, flatten, 0.9)], runs[(2, flatten, 0.9)]
    e1, e2 = _full(r1, "ema"), _full(r2, "ema")
    assert e1.keys() == e2.keys()
    m1 = [_full(r1, "masters", i) for i in range(STEPS + 1)]
    m2 = [_full(r2, "masters", i) for i in range(STEPS + 1)]
    for k in e1:
        diff = torch.stack([(a[k] - b[k]).abs() for a, b in zip(m1, m2)]).amax(0)
        _, b1 = ema64_and_bound(m1[0][k], [m[k] for m in m1[1:]], 0.9)
        _, b2 = ema64_and_bound(m2[0][k], [m[k] for m in m2[1:]], 0.9)
        assert bool(((e1[k] - e2[k]).abs().double() <= diff.double() + b1 + b2).all()), k
    # the runs really are the same training: the masters moved by up to lr = 1e-2 per step, and agree to 1e-3 (Adam's
    # normalised update turns reduction-order differences of small gradients into differences of up to lr)
    assert max(float((m1[-1][k] - m2[-1][k]).abs().max()) for k in e1) < 1e-3


# ------------------------------------------------------------------------------------------------
# checkpoints, consolidation, --init_from_full_ckpt, evaluation swap (W = 1, fp32 CPU)
# ------------------------------------------------------------------------------------------------
def _setup(ema=True, seed=1, decay=0.9):
    model = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=seed, model_ema=ema)
    opt = ShardedAdamW(model, lr=1e-2, weight_decay=0.1, model_ema_decay=decay if ema else None)
    return model, opt, get_warmup_cosine_scheduler(opt, 2, 100)


def _steps(model, opt, sched, start, stop):
    g = torch.Generator().manual_seed(99)
    batches = [(torch.randn(4, 3, 32, 32, generator=g), torch.randint(0, 10, (4,), generator=g)) for _ in range(stop)]
    for s in range(start, stop):
        model.forward_backward(*batches[s])
        model.clip_grad_norm_(1.0)
        opt.step()
        sched.step()


def _same(a, b):
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def test_checkpoint_gains_model_ema_only_with_the_flag_and_resume_restores_it(tmp_path, capsys):
    for ema in (False, True):
        model, opt, sched = _setup(ema)
        _steps(model, opt, sched, 0, 2)
        path = str(tmp_path / f"e{ema}.ckpt")
        save_ckpt(path, model, opt, sched)
        keys = set(torch.load(path, weights_only=False))
        assert keys == {"model", "shard_metadata", "optimizer", "lr_scheduler"} | ({"model_ema"} if ema else set())
    # uninterrupted 4 steps against 2 + resume + 2
    model, opt, sched = _setup()
    _steps(model, opt, sched, 0, 4)
    resumed, ropt, rsched = _setup(seed=5)
    load_ckpt(str(tmp_path / "eTrue.ckpt"), resumed, ropt, rsched)
    _steps(resumed, ropt, rsched, 2, 4)
    assert _same(resumed.ema_state_dict(), model.ema_state_dict())
    assert _same(resumed.state_dict(), model.state_dict())
    assert not _same(model.ema_state_dict(), model.state_dict())
    # a checkpoint without model_ema: the EMA starts from the restored weights, and says so
    capsys.readouterr()
    fallback, fopt, fsched = _setup(seed=6)
    load_ckpt(str(tmp_path / "eFalse.ckpt"), fallback, fopt, fsched)
    assert "the checkpoint has no model_ema: the model EMA starts from the restored weights" in capsys.readouterr().out
    assert _same(fallback.ema_state_dict(), fallback.state_dict())
    # a checkpoint with model_ema into a model without the flag: ignored
    plain, popt, psched = _setup(ema=False, seed=7)
    load_ckpt(str(tmp_path / "eTrue.ckpt"), plain, popt, psched)
    assert _same(plain.state_dict(), torch.load(str(tmp_path / "eTrue.ckpt"), weights_only=False)["model"])


def test_consolidation_writes_model_ema_and_init_from_full_reads_it(tmp_path):
    model, opt, sched = _setup()
    _steps(model, opt, sched, 0, 3)
    prefix = str(tmp_path / "epoch_1")
    save_ckpt(prefix + "_rank_0.ckpt", model, opt, sched)
    full = consolidate_files(prefix, save_path=prefix + "_full.pth")
    saved = torch.load(prefix + "_full.pth", weights_only=False)
    assert set(saved) == {"model", "shard_metadata", "model_ema"}
    assert _same(saved["model"], full) and saved["model_ema"].keys() == full.keys()
    # the consolidated EMA is the rank file's EMA, un-sharded
    fresh = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3, model_ema=True)
    fresh.load_full_state_dict(saved["model"])
    assert _same(fresh.ema_state_dict(), model.state_dict())  # without model_ema the EMA copies the loaded weights
    fresh.load_full_state_dict(saved["model_ema"], ema=True)
    assert _same(fresh.ema_state_dict(), model.ema_state_dict()) and _same(fresh.state_dict(), model.state_dict())
    # without the flag the file still loads (model_ema is not read)
    FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3).load_full_state_dict(saved["model"])
    with pytest.raises(RuntimeError, match="has no EMA"):
        FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3).load_full_state_dict(saved["model_ema"], ema=True)


def test_ema_evaluation_equals_a_model_loaded_with_the_consolidated_ema(tmp_path):
    model, opt, sched = _setup()
    _steps(model, opt, sched, 0, 3)
    prefix = str(tmp_path / "epoch_1")
    save_ckpt(prefix + "_rank_0.ckpt", model, opt, sched)
    consolidate_files(prefix, save_path=prefix + "_full.pth")
    ema_full = torch.load(prefix + "_full.pth", weights_only=False)["model_ema"]
    images = torch.randn(3, 3, 32, 32, generator=torch.Generator().manual_seed(5))
    model.eval()
    before = model(images)
    with model.ema_weights():
        got = model(images)
    after = model(images)
    loaded = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=11)
    loaded.load_full_state_dict(ema_full)
    assert torch.equal(got, loaded.eval()(images))
    assert torch.equal(before, after) and not torch.equal(got, before)


# ------------------------------------------------------------------------------------------------
# CLI: train two epochs with --model_ema, both accuracy lines, model_ema in the files, resume, init from full
# ------------------------------------------------------------------------------------------------
TINY = ["--fake_data", "--device", "cpu", "--nproc", "1", "--image_size", "32", "--patch_size", "8", "--embed_dim", "32",
        "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "4", "--warmup_steps", "2",
        "--lr", "1e-2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
        "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--model_ema", "--model_ema_decay", "0.9"]


def _run(args):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "run_vit_training.py", *args], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def test_cli_trains_evaluates_checkpoints_and_resumes_the_ema(tmp_path):
    ckpt = str(tmp_path / "c")
    out = _run([*TINY, "--ckpt_dir", ckpt, "--num_epochs", "2"])
    assert out.count("accuracy on val: ") == 2 and out.count("accuracy of the EMA on val: ") == 2
    assert "model_ema=True" in out and "model_ema_decay=0.9" in out
    e1 = torch.load(os.path.join(ckpt, "epoch_1_rank_0.ckpt"), weights_only=False)
    assert "model_ema" in e1 and e1["model_ema"].keys() == e1["model"].keys()
    uninterrupted = torch.load(os.path.join(ckpt, "epoch_2_rank_0.ckpt"), weights_only=False)
    assert not _same(uninterrupted["model_ema"], e1["model_ema"])
    out = _run([*TINY, "--ckpt_dir", ckpt, "--num_epochs", "2", "--resume_epoch", "1"])
    assert "resumed from checkpoint" in out and "accuracy of the EMA on val: " in out
    resumed = torch.load(os.path.join(ckpt, "epoch_2_rank_0.ckpt"), weights_only=False)
    assert _same(resumed["model_ema"], uninterrupted["model_ema"]) and _same(resumed["model"], uninterrupted["model"])
    consolidate_files(os.path.join(ckpt, "epoch_2"), save_path=os.path.join(ckpt, "full.pth"))
    out = _run([*TINY, "--ckpt_dir", str(tmp_path / "d"), "--num_epochs", "1", "--init_from_full_ckpt",
                os.path.join(ckpt, "full.pth")])
    assert "model EMA initialised from the checkpoint's model_ema" in out
    # the same file without --model_ema trains as before and prints no EMA line
    plain = [a for a in TINY if a not in ("--model_ema", "--model_ema_decay", "0.9")]
    out = _run([*plain, "--ckpt_dir", str(tmp_path / "e"), "--num_epochs", "1", "--init_from_full_ckpt",
                os.path.join(ckpt, "full.pth")])
    assert "accuracy on val: " in out and "EMA" not in out
    assert "model_ema" not in torch.load(os.path.join(str(tmp_path / "e"), "epoch_1_rank_0.ckpt"), weights_only=False)
