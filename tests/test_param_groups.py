"""Optimizer parameter groups (--filter_bias_and_norm / --layer_decay), on the CPU: the classification of every
parameter, the per-chunk group tables of every rank's shard, the CLI, checkpoints, FSDP equivalence on gloo and the
engine against PlainViT + torch.optim.AdamW with MAE-style parameter groups."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from param_groups_worker import launch
from helpers import ROOT, full_params_of, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.models.plain import PlainViT
from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW
from vit_10b_fsdp_example_b200.parallel import param_groups as pg
from vit_10b_fsdp_example_b200.parallel.layout import UnitLayout
from vit_10b_fsdp_example_b200.utils import get_warmup_cosine_scheduler

DINOV2_G = dict(embed_dim=1536, num_heads=24, num_blocks=40, mlp_ratio=4.0, class_token=True, reg_tokens=4,
                qk_norm=True, init_values=1e-5, swiglu=True)
BLOCK_DECAYED = {"attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight"}
TOKENS_CFG = dict(class_token=True, reg_tokens=2, qk_norm=True, init_values=0.5)


def all_groups(cfg):
    """timm name -> (layer id, decayed?) over the whole model, through the per-unit classifier."""
    out = {}
    for i in range(cfg.num_blocks):
        for p, v in pg.classify(cfg, f"blocks.{i}", vit.block_param_specs(cfg)).items():
            out[f"blocks.{i}.{p}"] = v
    out.update(pg.classify(cfg, "root", vit.root_param_specs(cfg)))
    return out


def expected_layer(name, L):
    """MAE get_layer_id_for_vit, written out independently."""
    m = re.match(r"blocks\.(\d+)\.", name)
    if m:
        return int(m.group(1)) + 1
    if name in ("cls_token", "reg_token", "pos_embed") or name.startswith("patch_embed"):
        return 0
    return L + 1


# ------------------------------------------------------------------------------------------------
# classification
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, DINOV2_G], ids=["vit10b", "dinov2_g"])
def test_decay_sets_and_layer_ids(kw):
    cfg = ViTConfig(**kw)
    groups = all_groups(cfg)
    L = cfg.num_blocks
    decayed = {n for n, (_, d) in groups.items() if d}
    want = {f"blocks.{i}.{p}" for i in range(L) for p in BLOCK_DECAYED} | {"patch_embed.proj.weight", "head.weight"}
    assert decayed == want
    no_decay = set(groups) - decayed
    for p in ("norm1.weight", "norm1.bias", "attn.qkv.bias", "attn.proj.bias", "norm2.weight", "norm2.bias",
              "mlp.fc1.bias", "mlp.fc2.bias"):
        assert f"blocks.{L - 1}.{p}" in no_decay
    assert {"pos_embed", "patch_embed.proj.bias", "norm.weight", "norm.bias", "head.bias"} <= no_decay
    if kw:
        assert {"cls_token", "reg_token", "blocks.3.ls1.gamma", "blocks.3.ls2.gamma", "blocks.0.attn.q_norm.weight",
                "blocks.0.attn.q_norm.bias", "blocks.0.attn.k_norm.weight", "blocks.0.attn.k_norm.bias"} <= no_decay
    for n, (lid, _) in groups.items():
        assert lid == expected_layer(n, L), n
    # every unit holds at most the 4 groups the kernel tables are sized for: a block 2, the root 4
    for d in (None, 0.75):
        assert len(pg.build_unit_groups(cfg, UnitLayout.build("root", vit.root_param_specs(cfg), 8, False), 0, 0.1, d,
                                        "cpu").rows) == 4


def test_lr_scales_against_the_formula():
    cfg = ViTConfig(**DINOV2_G)
    L, d = cfg.num_blocks, 0.75
    for n, (lid, dec) in all_groups(cfg).items():
        want = d ** (L + 1 - expected_layer(n, L))
        assert pg.lr_scale(lid, L, d) == pytest.approx(want, rel=1e-12), n
        assert pg.lr_scale(lid, L, None) == 1.0
    assert pg.lr_scale(L + 1, L, d) == 1.0 and pg.lr_scale(L, L, d) == d and pg.lr_scale(0, L, d) == d ** (L + 1)
    lay = UnitLayout.build("blocks.7", vit.block_param_specs(cfg), 4, False)
    ug = pg.build_unit_groups(cfg, lay, 1, 0.05, d, "cpu")
    rows = {(r.layer, r.decay): (r.lr_scale, r.weight_decay) for r in ug.rows}
    assert rows == {(8, False): (d ** (L - 7), 0.0), (8, True): (d ** (L - 7), 0.05)}
    assert torch.equal(ug.group_hyper, torch.tensor([[d ** (L - 7), 0.0], [d ** (L - 7), 0.05]], dtype=torch.float32))


def test_summary_counts_every_parameter_once():
    cfg = ViTConfig(**DINOV2_G)
    units = [pg.build_unit_groups(cfg, UnitLayout.build(n, specs, 1, True), 0, 0.1, 0.7, "cpu")
             for n, specs in [(f"blocks.{i}", vit.block_param_specs(cfg)) for i in range(cfg.num_blocks)]
             + [("root", vit.root_param_specs(cfg))]]
    rows = pg.summary(units)
    assert len(rows) == 2 * (cfg.num_blocks + 2)
    assert sum(r.elements for r in rows) == cfg.total_numel()
    assert sum(r.tensors for r in rows) == len(all_groups(cfg))
    text = pg.format_summary(rows)
    assert "layer_0_no_decay" in text and f"layer_{cfg.num_blocks + 1}_decay" in text


# ------------------------------------------------------------------------------------------------
# group tables of the shards
# ------------------------------------------------------------------------------------------------
def element_groups(lay, rank, param_group):
    """Group of every element of rank's shard (-1 = padding), rebuilt from UnitLayout.params / scatter_segments."""
    full = np.full(lay.full_numel, -1, dtype=np.int16)
    for p in lay.params:
        full[p.full_offset: p.full_offset + p.numel] = param_group[p.name]
    shard = np.full(lay.shard_numel, -1, dtype=np.int16)
    for full_off, shard_off, n in lay.scatter_segments(rank):
        shard[shard_off: shard_off + n] = full[full_off: full_off + n]
    return shard


@pytest.mark.parametrize("flatten", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("kw", [{}, TOKENS_CFG, dict(TOKENS_CFG, embed_dim=40, num_heads=5, num_classes=7)],
                         ids=["tiny", "tokens", "odd"])
def test_every_element_maps_to_its_parameters_group(kw, world, flatten):
    cfg = tiny_cfg(**kw)
    for name, specs in [("blocks.1", vit.block_param_specs(cfg)), ("root", vit.root_param_specs(cfg))]:
        lay = UnitLayout.build(name, specs, world, flatten)
        ug = pg.build_unit_groups(cfg, lay, 0, 0.1, 0.75, "cpu")
        keys = [(r.layer, r.decay) for r in ug.rows]
        cls = pg.classify(cfg, name, specs)
        param_group = {p: keys.index(k) for p, k in cls.items()}
        for rank in range(world):
            chunks = pg.build_chunk_groups(lay, rank, param_group)
            assert chunks.dtype == np.uint8 and chunks.size * 64 == lay.shard_numel
            eg = element_groups(lay, rank, param_group)
            real = eg >= 0
            assert np.array_equal(chunks[np.nonzero(real)[0] // 64], eg[real]), (name, rank)


def test_vit10b_root_tables_at_w8():
    cfg = ViTConfig()
    lay = UnitLayout.build("root", vit.root_param_specs(cfg), 8, False)
    ug = pg.build_unit_groups(cfg, lay, 0, 0.1, 0.75, "cpu")
    param_group = {p: [(r.layer, r.decay) for r in ug.rows].index(k)
                   for p, k in pg.classify(cfg, "root", vit.root_param_specs(cfg)).items()}
    for rank in (0, 5, 7):
        eg = element_groups(lay, rank, param_group)
        chunks = pg.build_chunk_groups(lay, rank, param_group)
        real = eg >= 0
        assert np.array_equal(chunks[np.nonzero(real)[0] // 64], eg[real])


def test_a_misaligned_layout_is_refused():
    lay = UnitLayout.build("blocks.0", [("a.weight", (64, 2)), ("a.bias", (64,))], 1, True)
    lay.params[1].full_offset = 100  # not a multiple of 64: a chunk would hold two parameters
    with pytest.raises(AssertionError, match="not a multiple of 64"):
        pg.build_chunk_groups(lay, 0, {"a.weight": 1, "a.bias": 0})


# ------------------------------------------------------------------------------------------------
# CLI and optimizer surface
# ------------------------------------------------------------------------------------------------
def test_cli_flags_and_validation():
    a = parse_args([])
    assert a.filter_bias_and_norm is False and a.layer_decay is None
    a = parse_args(["--filter_bias_and_norm", "--layer_decay", "0.75"])
    assert a.filter_bias_and_norm and a.layer_decay == 0.75
    assert parse_args(["--layer_decay", "1"]).layer_decay == 1.0
    for bad in ("0", "1.5", "nan", "-0.5", "inf"):
        with pytest.raises(SystemExit):
            parse_args(["--layer_decay", bad])


def test_optimizer_settings():
    model = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=0)
    plain = ShardedAdamW(model, lr=1e-3, weight_decay=0.1)
    assert plain.groups is None and plain.group_summary() is None
    g = plain.param_groups[0]
    assert g["filter_bias_and_norm"] is False and g["layer_decay"] is None
    lrd = ShardedAdamW(model, lr=1e-3, weight_decay=0.1, layer_decay=0.75)
    assert lrd.param_groups[0]["filter_bias_and_norm"] is True  # implied
    assert "filter_bias_and_norm=True, layer_decay=0.75" in repr(lrd)
    for bad in (0.0, 1.5, float("nan")):
        with pytest.raises(ValueError, match="layer_decay must be in"):
            ShardedAdamW(model, layer_decay=bad)
    ug = lrd.groups["root"]
    assert ug.chunk_groups.dtype == torch.uint8 and ug.chunk_groups.numel() * 64 == model.root.layout.shard_numel


# ------------------------------------------------------------------------------------------------
# checkpoints
# ------------------------------------------------------------------------------------------------
def _opt(model, **kw):
    return ShardedAdamW(model, lr=1e-3, weight_decay=0.1, **kw)


def test_state_dict_round_trip_and_refusals():
    model = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=0)
    sd = _opt(model, layer_decay=0.75).state_dict()
    assert sd["param_groups"][0]["layer_decay"] == 0.75 and sd["param_groups"][0]["filter_bias_and_norm"] is True
    o = _opt(model, layer_decay=0.75)
    o.load_state_dict(sd)
    assert o.param_groups[0]["layer_decay"] == 0.75
    with pytest.raises(ValueError, match="pass --layer_decay 0.75"):
        _opt(model).load_state_dict(sd)
    with pytest.raises(ValueError, match="pass --layer_decay 0.75"):
        _opt(model, filter_bias_and_norm=True).load_state_dict(sd)
    with pytest.raises(ValueError, match="pass --layer_decay 0.75"):
        _opt(model, layer_decay=0.5).load_state_dict(sd)
    filt = _opt(model, filter_bias_and_norm=True).state_dict()
    with pytest.raises(ValueError, match="pass --filter_bias_and_norm"):
        _opt(model).load_state_dict(filt)
    with pytest.raises(ValueError, match="drop --layer_decay"):
        _opt(model, layer_decay=0.75).load_state_dict(filt)
    old = _opt(model).state_dict()
    for g in old["param_groups"]:  # written before parameter groups existed
        del g["filter_bias_and_norm"], g["layer_decay"]
    _opt(model).load_state_dict(old)
    with pytest.raises(ValueError, match="drop --filter_bias_and_norm"):
        _opt(model, filter_bias_and_norm=True).load_state_dict(old)


def test_restored_weight_decay_reaches_the_tables():
    model = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=0)
    sd = ShardedAdamW(model, lr=1e-3, weight_decay=0.05, filter_bias_and_norm=True).state_dict()
    o = ShardedAdamW(model, lr=1e-3, weight_decay=0.1, filter_bias_and_norm=True)
    o.load_state_dict(sd)
    for ug in o.groups.values():
        assert {round(x, 6) for x in ug.group_hyper[:, 1].tolist()} == {0.0, 0.05}


def _cli(args, ok=True):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "run_vit_training.py", *args], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=300)
    assert (r.returncode == 0) == ok, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout + r.stderr


CLI = ["--fake_data", "--device", "cpu", "--nproc", "1", "--image_size", "28", "--patch_size", "14", "--embed_dim", "32",
       "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "4", "--warmup_steps", "1",
       "--max_steps", "2", "--num_workers", "0", "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1",
       "--class_token", "--init_values", "1e-5"]


def test_cli_logs_groups_checkpoints_and_resumes(tmp_path):
    ck = ["--ckpt_dir", str(tmp_path)]
    out = _cli([*CLI, *ck, "--num_epochs", "1", "--layer_decay", "0.75"])
    assert "=== parameter groups ===" in out and "layer_0_no_decay: lr_scale 0.421875" in out
    assert "layer_3_decay: lr_scale 1, weight_decay 0.1, 1 tensors" in out
    out = _cli([*CLI, *ck, "--num_epochs", "2", "--resume_epoch", "1"], ok=False)
    assert "pass --layer_decay 0.75 to resume it" in out
    out = _cli([*CLI, *ck, "--num_epochs", "2", "--resume_epoch", "1", "--layer_decay", "0.75"])
    assert "resumed from checkpoint" in out and "epoch 2 step 1" in out and "training completed" in out
    off = _cli([*CLI, "--ckpt_dir", str(tmp_path / "off"), "--num_epochs", "1"])
    assert "=== parameter groups ===" not in off


# ------------------------------------------------------------------------------------------------
# FSDP equivalence (gloo) and the torch.optim.AdamW reference
# ------------------------------------------------------------------------------------------------
GROUPED = {"layer_decay": 0.75, "model": TOKENS_CFG}


@pytest.fixture(scope="module")
def grouped_baseline(tmp_path_factory):
    return launch(1, dict(GROUPED, steps=4), str(tmp_path_factory.mktemp("pg") / "r.json"))


def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.mark.parametrize("world,flatten,no_fsdp", [(1, True, False), (2, False, False), (2, True, False),
                                                   (4, False, False), (4, True, False), (8, False, False),
                                                   (8, True, False), (2, False, True)])
def test_sharded_runs_reproduce_one_process(world, flatten, no_fsdp, grouped_baseline, tmp_path):
    res = launch(world, dict(GROUPED, steps=4, flatten=flatten, no_fsdp=no_fsdp), str(tmp_path / "r.json"))
    _close(res["losses"], grouped_baseline["losses"])
    _close(res["norms"], grouped_baseline["norms"], tol=1e-4)


def test_groups_change_the_trajectory(grouped_baseline, tmp_path):
    plain = launch(1, {"model": TOKENS_CFG, "steps": 4}, str(tmp_path / "r.json"))
    assert abs(plain["losses"][-1] - grouped_baseline["losses"][-1]) > 1e-4


def mae_param_groups(plain, base_lr, wd, layer_decay):
    """MAE param_groups_lrd, written against PlainViT's named_parameters: one group per (layer, decay) pair."""
    L = plain.cfg.num_blocks
    groups = {}
    for n, p in plain.named_parameters():
        no_decay = p.ndim <= 1 or n in ("pos_embed", "cls_token", "reg_token")
        lid = expected_layer(n, L)
        g = groups.setdefault((lid, no_decay), {"params": [], "weight_decay": 0.0 if no_decay else wd,
                                                "lr_scale": layer_decay ** (L + 1 - lid)})
        g["params"].append(p)
    for g in groups.values():
        g["lr"] = base_lr * g["lr_scale"]
    return list(groups.values())


@pytest.mark.parametrize("kw", [{}, TOKENS_CFG], ids=["plain", "tokens"])
def test_engine_matches_torch_adamw_with_mae_groups(kw):
    cfg = tiny_cfg(**kw)
    d, wd, steps = 0.5, 0.3, 5
    model = FSDPViT(cfg, dtype=torch.float32, seed=3)
    opt = ShardedAdamW(model, lr=3e-3, weight_decay=wd, layer_decay=d)
    sched = get_warmup_cosine_scheduler(opt, 2, 10)
    plain = PlainViT(cfg).train()
    sd = full_params_of(model)
    for k, shape in vit.logical_shapes(cfg).items():
        sd[k] = sd[k][:, : cfg.patch_k].reshape(shape) if k == "patch_embed.proj.weight" else sd[k].reshape(shape)
    plain.load_state_dict(sd, strict=True)
    ref = torch.optim.AdamW(mae_param_groups(plain, opt.param_groups[0]["lr"], wd, d), lr=1.0)
    g = torch.Generator().manual_seed(0)
    for s in range(steps):
        images = torch.randn(4, 3, cfg.image_size, cfg.image_size, generator=g)
        target = torch.randint(0, cfg.num_classes, (4,), generator=g)
        for rg in ref.param_groups:
            rg["lr"] = opt.param_groups[0]["lr"] * rg["lr_scale"]
        loss = model.forward_backward(images, target)
        opt.step()
        sched.step()
        ref.zero_grad()
        ref_loss = torch.nn.functional.cross_entropy(plain(images), target)
        ref_loss.backward()
        ref.step()
        assert abs(loss.item() - ref_loss.item()) <= 1e-5 * max(1.0, abs(ref_loss.item())), s
    got = full_params_of(model)
    D = cfg.embed_dim
    for k, v in plain.state_dict().items():
        e = (got[k][:, : cfg.patch_k] if k == "patch_embed.proj.weight" else got[k]).reshape(v.shape)
        # the key bias (qkv.bias[D:2D], k_norm.bias) cannot change the softmax: its true gradient is 0, both sides get
        # rounding noise, and Adam turns the noise's sign into a full +-lr step
        if k.endswith("k_norm.bias"):
            continue
        if k.endswith("attn.qkv.bias"):
            e, v = torch.cat([e[:D], e[2 * D:]]), torch.cat([v[:D], v[2 * D:]])
        torch.testing.assert_close(e, v, rtol=1e-5, atol=1e-6, msg=k)
