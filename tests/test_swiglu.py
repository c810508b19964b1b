"""SwiGLU MLP (--swiglu): the torch_ops reference of the gated forward and its gradient against fp64, the engine
against an fp64 autograd oracle written in timm's GluMlp form, parameters, the CLI, FSDP equivalence, checkpoints
(timm-layout state dicts and the refusals), the AG-fusion exclusion and the build of the sm_90a kernels.

The oracle follows timm's SwiGLUPacked = GluMlp(act_layer=nn.SiLU, gate_last=False) literally: u = fc1(x),
(gate, value) = u.chunk(2, -1), g = drop1(silu(gate) * value), norm = Identity, fc2(g), drop2."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from dist_worker import launch
from helpers import full_grads_of, full_params_of, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IMAGES = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(7))
TARGET = torch.tensor([1, 5, 7, 2])


def sw_cfg(**kw):
    return tiny_cfg(**dict(dict(swiglu=True), **kw))


def randomize(model, seed=0):
    """Prefix tokens, LayerScale and QK-norm parameters at magnitudes that move the loss."""
    g = torch.Generator().manual_seed(seed)
    full = full_params_of(model)
    for k, v in full.items():
        if k in ("cls_token", "reg_token"):
            full[k] = torch.randn(v.shape, generator=g)
        elif k.endswith(("ls1.gamma", "ls2.gamma")):
            sign = torch.where(torch.rand(v.shape, generator=g) < 0.5, -1.0, 1.0)
            full[k] = sign * (0.5 + torch.rand(v.shape, generator=g))
        elif ".q_norm." in k or ".k_norm." in k:
            full[k] = (1.0 if k.endswith("weight") else 0.0) + 0.5 * torch.randn(v.shape, generator=g)
    model.load_full_state_dict(full)


# ------------------------------------------------------------------------------------------------
# the ops against fp64
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,K,Hd", [(7, 8, 16), (33, 24, 48), (5, 40, 208)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ops_against_fp64(M, K, Hd, dtype):
    g = torch.Generator().manual_seed(M + K + Hd)
    x = (torch.randn(M, K, generator=g) * 2).to(dtype)
    w = torch.randn(Hd, K, generator=g).to(dtype)
    b = torch.randn(Hd, generator=g).to(dtype)
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -23

    xx, ww, bb = (t.double().requires_grad_(True) for t in (x, w, b))
    u64 = F.linear(xx, ww, bb)
    gate, value = u64.chunk(2, dim=-1)
    g64 = F.silu(gate) * value
    out, pre = torch_ops.linear_fwd(x, w, b, act="swiglu", want_preact=True)
    assert out.shape == (M, Hd // 2) and pre.shape == (M, Hd) and out.dtype == dtype
    tol = lambda ref: 2 * ulp * ref.abs() + 1e-4 * ref.abs().max()  # noqa: E731  one rounding + fp32 sums
    assert ((out.double() - g64).abs() <= tol(g64)).all()
    assert ((pre.double() - u64).abs() <= tol(u64)).all()
    assert torch.equal(torch_ops.swiglu_fwd(pre), torch_ops.swiglu_fwd(pre.clone()))
    assert ((torch_ops.swiglu_fwd(pre).double() - torch_ops._swiglu(pre.double())).abs()
            <= tol(torch_ops._swiglu(pre.double()))).all()

    # backward through fc2: dh = dy w2, du = d(silu(gate) * value) / du, against autograd
    D = 9
    w2 = torch.randn(D, Hd // 2, generator=g).to(dtype)
    dy = torch.randn(M, D, generator=g).to(dtype)
    u_in = pre.double().requires_grad_(True)
    ga, va = u_in.chunk(2, dim=-1)
    (F.linear(F.silu(ga) * va, w2.double()) * dy.double()).sum().backward()
    du, cs = torch_ops.linear_dgrad(dy, w2, dswiglu_preact=pre, want_colsum=True)
    assert du.shape == (M, Hd) and du.dtype == dtype
    assert ((du.double() - u_in.grad).abs() <= tol(u_in.grad)).all()
    assert torch.allclose(cs.double(), du.double().sum(0), rtol=1e-5, atol=1e-5)
    dh = torch_ops.linear_dgrad(dy, w2)
    du2 = torch_ops.swiglu_bwd(dh, pre)
    assert ((du2.double() - u_in.grad).abs() <= 2 * tol(u_in.grad)).all()


def test_swiglu_refuses_a_residual_or_row_scale():
    x, w = torch.randn(4, 8), torch.randn(16, 8)
    with pytest.raises(AssertionError, match="swiglu: no residual or row scale"):
        torch_ops.linear_fwd(x, w, act="swiglu", residual=torch.randn(4, 8))


# ------------------------------------------------------------------------------------------------
# the engine against the fp64 oracle
# ------------------------------------------------------------------------------------------------
def autograd_vit_loss_glu(cfg, params, images, target, masks=None, pos_mask=None, soft=None):
    """timm VisionTransformer(mlp_layer=SwiGLUPacked, act_layer=nn.SiLU) with the optional prefix tokens, QK norm,
    LayerScale, dropout / drop-path factors (masks: per-block dict {"att", "proj", "fc1", "fc2", "sa", "sm"}), a
    pos-dropout factor and soft targets."""
    B = images.shape[0]
    N, T, D, H, hd, ps = cfg.num_patches, cfg.num_tokens, cfg.embed_dim, cfg.num_heads, cfg.head_dim, cfg.patch_size
    w = params["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(D, 3, ps, ps)
    x = F.conv2d(images, w, params["patch_embed.proj.bias"], stride=ps).flatten(2).transpose(1, 2)
    pos = params["pos_embed"].view(1, cfg.pos_len, D)
    if cfg.class_token:
        prefix = [params["cls_token"].view(1, 1, D).expand(B, -1, -1)]
        if cfg.reg_tokens:
            prefix.append(params["reg_token"].view(1, -1, D).expand(B, -1, -1))
        x = torch.cat(prefix + [x + pos], dim=1) if cfg.no_embed_class else torch.cat(prefix + [x], dim=1) + pos
    else:
        x = x + pos
    if pos_mask is not None:
        x = x * pos_mask
    for i in range(cfg.num_blocks):
        g = lambda n: params[f"blocks.{i}.{n}"]  # noqa: E731
        mk = (masks or [None] * cfg.num_blocks)[i] or {}
        m = lambda name, t: t * mk[name] if name in mk else t  # noqa: E731
        ls = lambda n, t: g(n) * t if cfg.init_values else t  # noqa: E731
        h = F.layer_norm(x, (D,), g("norm1.weight"), g("norm1.bias"), 1e-5)
        q, k, v = F.linear(h, g("attn.qkv.weight"), g("attn.qkv.bias")).reshape(B, T, 3, H, hd).permute(2, 0, 3, 1, 4)
        if cfg.qk_norm:
            q = F.layer_norm(q, (hd,), g("attn.q_norm.weight"), g("attn.q_norm.bias"), 1e-5)
            k = F.layer_norm(k, (hd,), g("attn.k_norm.weight"), g("attn.k_norm.bias"), 1e-5)
        att = m("att", ((q @ k.transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1))
        a = (att @ v).transpose(1, 2).reshape(B, T, D)
        x = x + ls("ls1.gamma", m("sa", m("proj", F.linear(a, g("attn.proj.weight"), g("attn.proj.bias")))))
        h = F.layer_norm(x, (D,), g("norm2.weight"), g("norm2.bias"), 1e-5)
        gate, value = F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias")).chunk(2, dim=-1)  # GluMlp, gate first
        h = m("fc1", F.silu(gate) * value)  # drop1; GluMlp.norm is Identity
        x = x + ls("ls2.gamma", m("sm", m("fc2", F.linear(h, g("mlp.fc2.weight"), g("mlp.fc2.bias")))))
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x[:, 0] if cfg.class_token else x.mean(dim=1), params["head.weight"], params["head.bias"])
    if soft is not None:
        return (-soft.double() * torch.log_softmax(logits, dim=-1)).sum(-1).mean(), logits
    return F.cross_entropy(logits, target), logits


def _check_against_oracle(model, images, target, **kw):
    loss = model.forward_backward(images, target)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    assert params["blocks.0.mlp.fc2.weight"].shape == (model.cfg.embed_dim, model.cfg.hidden_dim // 2)
    ref_loss, ref_logits = autograd_vit_loss_glu(model.cfg, params, images.double(), target, **kw)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 1e-5, (loss.item(), ref_loss.item())
    for name, p in params.items():
        g = p.grad if p.grad is not None else torch.zeros_like(p)
        err = (got[name].double() - g.view(got[name].shape)).abs().max().item()
        if name.endswith("k_norm.bias"):  # exactly zero: the softmax cancels q . b_k; fp32 rounding is left
            assert g.abs().max().item() < 1e-12 and err < 1e-7, f"{name}: err {err}"
            continue
        scale = g.abs().max().item() + 1e-8
        assert err / scale < 2e-4, f"{name}: err {err} scale {scale}"
    return ref_logits


VARIANTS = [dict(), dict(qk_norm=True), dict(init_values=1e-5), dict(class_token=True, reg_tokens=4),
            dict(class_token=True, reg_tokens=4, init_values=1e-5, qk_norm=True, no_embed_class=True)]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("grad_ckpt,keep,flatten", [(True, 0, False), (False, 0, False), (True, 0, True),
                                                    (True, 1, False), (True, 99, True)])
def test_engine_matches_autograd(variant, grad_ckpt, keep, flatten):
    cfg = sw_cfg(**variant)
    model = FSDPViT(cfg, dtype=torch.float32, grad_ckpt=grad_ckpt, ckpt_keep_blocks=keep, flatten_parameters=flatten,
                    seed=3)
    randomize(model)
    images = torch.randn(4, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(1))
    ref_logits = _check_against_oracle(model, images, TARGET)
    assert torch.allclose(model.eval()(images).double(), ref_logits.detach(), atol=1e-4)


@pytest.mark.parametrize("extras", [{"P": 99, "h": 99, "g": 99}, {"P": 1, "h": 0, "g": 1}, {"P": 0, "h": 2, "g": 0}])
def test_kept_blocks_with_extras_match_autograd(extras):
    model = FSDPViT(sw_cfg(class_token=True, reg_tokens=3), dtype=torch.float32, grad_ckpt=True, ckpt_keep_blocks=99,
                    seed=3)
    model.keep_extras = extras
    randomize(model, seed=1)
    _check_against_oracle(model, IMAGES, TARGET)


@pytest.mark.parametrize("kw", [dict(), dict(qk_norm=True), dict(init_values=1e-5, qk_norm=True, class_token=True,
                                                                 reg_tokens=4)])
def test_flash_style_path_matches_autograd(monkeypatch, kw):
    monkeypatch.setattr(torch_ops, "FLASH_ATTENTION", True)
    for mode in (dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)):
        model = FSDPViT(sw_cfg(**kw), dtype=torch.float32, seed=3, **mode)
        randomize(model, seed=2)
        _check_against_oracle(model, IMAGES, TARGET)


def _model_masks(model, B):
    """The multiplicative dropout / drop-path factors the model's blocks draw in its next training step."""
    cfg, ctx = model.cfg, model.drop
    T, H, D = cfg.num_tokens, cfg.num_heads, cfg.embed_dim
    pa, pm = cfg.att_dropout, cfg.mlp_dropout
    out = []
    for i, rate in enumerate(vit.drop_path_rates(cfg)):
        site = i * 8
        m = {}
        if pa > 0:
            m["att"] = torch_ops.dropout(torch.ones(B * H, T, T, dtype=torch.float64), pa,
                                         ctx.key(site)).view(B, H, T, T)
        if pm > 0:
            m["proj"] = torch_ops.dropout(torch.ones(B * T, D, dtype=torch.float64), pm,
                                          ctx.key(site + 1)).view(B, T, D)
            # drop1 acts on g = silu(gate) * value: [T, Hd / 2]
            m["fc1"] = torch_ops.dropout(torch.ones(B * T, cfg.hidden_dim // 2, dtype=torch.float64), pm,
                                         ctx.key(site + 2)).view(B, T, -1)
            m["fc2"] = torch_ops.dropout(torch.ones(B * T, D, dtype=torch.float64), pm, ctx.key(site + 3)).view(B, T, D)
        if rate > 0:
            for name, off in (("sa", 4), ("sm", 5)):
                m[name] = torch_ops.drop_path_scale(ctx.key(site + off), rate, B, model.rank * B,
                                                    "cpu").double().view(B, 1, 1)
        out.append(m)
    pos_mask = None
    if cfg.pos_dropout > 0:
        pos_mask = torch_ops.dropout(torch.ones(B * T, D, dtype=torch.float64), cfg.pos_dropout,
                                     ctx.key(7_000_001)).view(B, T, D)
    return out, pos_mask


@pytest.mark.parametrize("kw", [dict(att_dropout=0.2), dict(mlp_dropout=0.2), dict(pos_dropout=0.3),
                                dict(drop_path_rate=0.5, init_values=1e-5, qk_norm=True),
                                dict(att_dropout=0.1, mlp_dropout=0.1, pos_dropout=0.1, drop_path_rate=0.5,
                                     class_token=True, reg_tokens=2)])
@pytest.mark.parametrize("mode", [dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)])
def test_composes_with_dropout_and_drop_path(kw, mode):
    cfg = sw_cfg(num_blocks=4, **kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3, **mode)
    randomize(model, seed=3)
    images = torch.randn(8, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(2))
    target = torch.randint(0, 10, (8,), generator=torch.Generator().manual_seed(2))
    masks, pos_mask = _model_masks(model, 8)
    _check_against_oracle(model, images, target, masks=masks, pos_mask=pos_mask)


@pytest.mark.parametrize("kw", [dict(mixup=0.8, smoothing=0.1), dict(cutmix=1.0, smoothing=0.1, class_token=True)])
def test_mixup_and_smoothing_match_autograd(kw):
    cfg = sw_cfg(**kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3)
    randomize(model, seed=4)
    mix = vit.draw_mix(cfg, vit.mix_rng(model.drop.seed, model.step_count, model.rank))
    assert mix is not None
    mixed = torch_ops.mix_images(IMAGES, mix)
    soft = torch_ops.mixup_target(TARGET, cfg.num_classes, mix[0], cfg.smoothing)
    loss = model.forward_backward(IMAGES, TARGET)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    ref_loss, _ = autograd_vit_loss_glu(cfg, params, mixed.double(), TARGET, soft=soft)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 1e-5, (loss.item(), ref_loss.item())
    for name, p in params.items():
        err = (got[name].double() - p.grad.view(got[name].shape)).abs().max().item()
        assert err / (p.grad.abs().max().item() + 1e-8) < 2e-4, name


# ------------------------------------------------------------------------------------------------
# default behaviour, parameters, config
# ------------------------------------------------------------------------------------------------
def test_flag_off_calls_nothing_new(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("SwiGLU op called without --swiglu")

    monkeypatch.setattr(torch_ops, "swiglu_fwd", boom)
    monkeypatch.setattr(torch_ops, "swiglu_bwd", boom)
    monkeypatch.setattr(torch_ops, "_swiglu", boom)
    monkeypatch.setattr(torch_ops, "_dswiglu", boom)
    for kw in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
        model = FSDPViT(tiny_cfg(mlp_dropout=0.1, drop_path_rate=0.3), dtype=torch.float32, seed=3, **kw)
        model.forward_backward(IMAGES, TARGET)
        model.eval()(IMAGES)
    assert dict(vit.block_param_specs(tiny_cfg()))["mlp.fc2.weight"] == (64, 128)


def test_parameters_order_init_and_counts():
    cfg, base = sw_cfg(), tiny_cfg()
    D, Hd = cfg.embed_dim, cfg.hidden_dim
    specs, bspecs = vit.block_param_specs(cfg), vit.block_param_specs(base)
    assert [n for n, _ in specs] == [n for n, _ in bspecs]  # timm's names and order
    assert dict(specs)["mlp.fc1.weight"] == (Hd, D) and dict(specs)["mlp.fc1.bias"] == (Hd,)
    assert dict(specs)["mlp.fc2.weight"] == (D, Hd // 2) and dict(specs)["mlp.fc2.bias"] == (D,)
    assert cfg.mlp_out_dim == Hd // 2 and base.mlp_out_dim == Hd
    assert cfg.block_numel() == sum(torch.Size(s).numel() for _, s in specs)
    assert base.block_numel() - cfg.block_numel() == D * Hd // 2
    a = full_params_of(FSDPViT(cfg, dtype=torch.float32, seed=5))
    b = full_params_of(FSDPViT(base, dtype=torch.float32, seed=5))
    assert set(a) == set(b)
    # same draw order: everything up to fc1 is the same draw; fc2's U(+-1/sqrt(fan_in)) has fan_in Hd / 2
    for k in b:
        if k.endswith(("mlp.fc2.weight", "mlp.fc2.bias")) or (k.startswith("blocks.") and not k.startswith("blocks.0.")) \
                or not k.startswith("blocks."):
            continue
        assert torch.equal(a[k], b[k]), k
    bound = 1.0 / (Hd // 2) ** 0.5
    w2 = a["blocks.0.mlp.fc2.weight"]
    assert w2.abs().max() <= bound and w2.abs().max() > 0.9 * bound
    # DINOv2-g: Hd = int(1536 * 5.33334) = 8192, H' = 4096
    g = ViTConfig(embed_dim=1536, num_heads=24, mlp_ratio=2.66667 * 2, swiglu=True, class_token=True, reg_tokens=4,
                  init_values=1e-5)
    assert (g.hidden_dim, g.mlp_out_dim) == (8192, 4096)
    assert dict(vit.block_param_specs(g))["mlp.fc2.weight"] == (1536, 4096)


def test_flops_and_extra_bytes():
    c, c0 = ViTConfig(swiglu=True), ViTConfig()
    D, Hd, T, L = c.embed_dim, c.hidden_dim, c.num_tokens, c.num_blocks
    assert c0.flops_per_image() - c.flops_per_image() == 4.0 * L * 2 * T * D * (Hd // 2)
    per_block = 2 * T * (3 * D * D + D * D + D * Hd + D * Hd // 2) + 4 * T * T * D
    assert c.flops_per_image() == 4.0 * (L * per_block + 2 * c.num_patches * c.patch_k * D + 2 * D * c.num_classes)
    a = FSDPViT(sw_cfg(), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    assert a.lean_bytes_per_block(4) == b.lean_bytes_per_block(4)  # u is [T, Hd] in both forms
    ea, eb = dict(a.extra_bytes_per_block(4)), dict(b.extra_bytes_per_block(4))
    unit = 4 * a.cfg.num_tokens * a.cfg.embed_dim * 4
    assert eb["g"] == int(a.cfg.mlp_ratio * unit) and ea["g"] == int(a.cfg.mlp_ratio / 2 * unit)
    assert ea["P"] == eb["P"] and ea["h"] == eb["h"]


def test_cli_parsing_and_rejections():
    assert parse_args([]).swiglu is False and ViTConfig.from_args(parse_args([])).swiglu is False
    c = ViTConfig.from_args(parse_args(["--swiglu", "--embed_dim", "1536", "--num_heads", "24", "--mlp_ratio",
                                        "5.33334"]))
    assert c.swiglu and (c.hidden_dim, c.mlp_out_dim) == (8192, 4096)
    with pytest.raises(SystemExit):
        parse_args(["--swiglu", "--embed_dim", "100", "--num_heads", "2", "--mlp_ratio", "1.5"])  # Hd = 150
    with pytest.raises(ValueError, match=r"--swiglu needs the MLP width Hd = int\(embed_dim \* mlp_ratio\) to be a "
                                         r"multiple of 16.*got Hd = 136"):
        sw_cfg(embed_dim=68, mlp_ratio=2.0)
    parse_args(["--embed_dim", "100", "--num_heads", "2", "--mlp_ratio", "1.5"])  # without the flag: no such rule
    tiny_cfg(embed_dim=68, mlp_ratio=2.0)


def test_cli_refusal_message():
    r = subprocess.run([sys.executable, "run_vit_training.py", "--swiglu", "--embed_dim", "100", "--num_heads", "2",
                        "--mlp_ratio", "1.5"], cwd=ROOT, capture_output=True, text=True, timeout=120)
    assert r.returncode != 0 and "multiple of 16" in r.stderr and "Hd = 150" in r.stderr


def test_fusable_params_leave_a_swiglu_fc1_to_the_unit_gather():
    from vit_10b_fsdp_example_b200.parallel.backends import Sm100Backend
    from vit_10b_fsdp_example_b200.parallel.layout import UnitLayout

    be = Sm100Backend.__new__(Sm100Backend)
    be.world = 2
    for cfg, want in ((tiny_cfg(), ("attn.qkv.weight", "mlp.fc1.weight")), (sw_cfg(), ("attn.qkv.weight",))):
        lay = UnitLayout.build("blocks.0", vit.block_param_specs(cfg), world=2, flatten=False)
        assert be.fusable_params(lay) == want


# ------------------------------------------------------------------------------------------------
# FSDP equivalence and checkpoints
# ------------------------------------------------------------------------------------------------
MODEL = {"swiglu": True, "class_token": True, "reg_tokens": 2, "init_values": 1e-5}


@pytest.fixture(scope="module")
def sw_baseline(tmp_path_factory):
    out = tmp_path_factory.mktemp("sw_base") / "r.json"
    return launch(1, {"model": MODEL, "steps": 4}, str(out))


def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.mark.parametrize("opts", [{}, {"flatten": True}])
def test_two_ranks_reproduce_one(opts, sw_baseline, tmp_path):
    res = launch(2, dict(opts, model=MODEL, steps=4), str(tmp_path / "r.json"))
    _close(res["losses"], sw_baseline["losses"])
    _close(res["norms"], sw_baseline["norms"], tol=1e-4)


def test_resume_equals_uninterrupted(tmp_path):
    d = str(tmp_path)
    model = dict(MODEL, mlp_dropout=0.1)
    full = launch(2, {"model": model, "steps": 5}, os.path.join(d, "full.json"))
    launch(2, {"model": model, "steps": 3, "save_at": 3, "save_path": os.path.join(d, "e1_rank_{rank}.ckpt")},
           os.path.join(d, "part.json"))
    rest = launch(2, {"model": model, "steps": 5, "resume_from": os.path.join(d, "e1_rank_{rank}.ckpt"),
                      "resume_step": 3}, os.path.join(d, "rest.json"))
    for a, b in zip(rest["losses"], full["losses"][3:]):
        assert abs(a - b) < 1e-6


def test_shard_metadata_records_the_flag():
    assert FSDPViT(sw_cfg(), dtype=torch.float32, seed=1).get_shard_metadata()["model"]["swiglu"] is True
    assert FSDPViT(tiny_cfg(), dtype=torch.float32, seed=1).get_shard_metadata()["model"]["swiglu"] is False


def test_consolidated_checkpoint_loads_into_plain_vit_and_back(tmp_path):
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    d = str(tmp_path)
    prefix = os.path.join(d, "epoch_1")
    launch(2, {"model": MODEL, "steps": 2, "seed": 7, "dump_state": prefix + "_rank_{rank}.ckpt"},
           os.path.join(d, "r.json"))
    full = consolidate_files(prefix, save_path=prefix + "_full.pth")
    cfg = tiny_cfg(**MODEL)
    D, Hd = cfg.embed_dim, cfg.hidden_dim
    assert full["blocks.0.mlp.fc1.weight"].shape == (Hd, D) and full["blocks.0.mlp.fc2.weight"].shape == (D, Hd // 2)
    images = torch.randn(3, 3, cfg.image_size, cfg.image_size)
    engine = FSDPViT(cfg, dtype=torch.float32, seed=99)
    engine.load_full_state_dict(full)
    plain = PlainViT.from_consolidated(prefix + "_full.pth", cfg).eval()
    assert set(plain.state_dict()) == set(full)
    assert type(plain.blocks[0].mlp).__name__ == "_GluMlp"
    with torch.no_grad():
        assert torch.allclose(engine.eval()(images), plain(images), atol=1e-4)
    randomize(engine, seed=5)
    sd = full_params_of(engine)
    for k, shape in vit.logical_shapes(cfg).items():
        sd[k] = sd[k][:, : cfg.patch_k].reshape(shape) if k == "patch_embed.proj.weight" else sd[k].reshape(shape)
    plain.load_state_dict(sd, strict=True)
    with torch.no_grad():
        want = plain(images)
    assert torch.allclose(engine.eval()(images), want, atol=1e-4)
    back = FSDPViT(cfg, dtype=torch.float32, seed=5)
    back.load_full_state_dict(plain.state_dict())
    assert torch.allclose(back.eval()(images), want, atol=1e-4)


def _cli(args, ok=True):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "run_vit_training.py", *args], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=300)
    assert (r.returncode == 0) == ok, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout + r.stderr


COMMON = ["--fake_data", "--device", "cpu", "--nproc", "1", "--image_size", "28", "--patch_size", "14",
          "--embed_dim", "32", "--num_heads", "2", "--num_blocks", "1", "--num_classes", "10", "--batch_size", "4",
          "--warmup_steps", "1", "--max_steps", "1", "--num_workers", "0", "--num_epochs", "1",
          "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--lr", "0", "--weight_decay", "0"]


def test_timm_reg4_dinov2_layout_state_dict_loads(tmp_path):
    """A hand-built timm *_reg4_dinov2-layout state dict (cls_token, 4 reg_token, pos_embed over the patches only,
    LayerScale, SwiGLUPacked MLP: fc1 [Hd, D], fc2 [D, Hd / 2]) starts a run through the CLI and arrives verbatim."""
    D, Hd, Ps = 32, 96, 14  # mlp_ratio 3: Hd = 96, H' = 48
    sd = {"cls_token": (1, 1, D), "reg_token": (1, 4, D), "pos_embed": (1, 4, D),
          "patch_embed.proj.weight": (D, 3, Ps, Ps), "patch_embed.proj.bias": (D,),
          "norm.weight": (D,), "norm.bias": (D,), "head.weight": (10, D), "head.bias": (10,)}
    blk = {"norm1.weight": (D,), "norm1.bias": (D,), "attn.qkv.weight": (3 * D, D), "attn.qkv.bias": (3 * D,),
           "attn.proj.weight": (D, D), "attn.proj.bias": (D,), "ls1.gamma": (D,), "norm2.weight": (D,),
           "norm2.bias": (D,), "mlp.fc1.weight": (Hd, D), "mlp.fc1.bias": (Hd,), "mlp.fc2.weight": (D, Hd // 2),
           "mlp.fc2.bias": (D,), "ls2.gamma": (D,)}
    sd.update({f"blocks.0.{k}": v for k, v in blk.items()})
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(s, generator=g) for k, s in sd.items()}
    path = str(tmp_path / "dinov2.pth")
    torch.save(sd, path)
    flags = ["--mlp_ratio", "3", "--class_token", "--reg_tokens", "4", "--no_embed_class", "--init_values", "1e-5"]
    _cli([*COMMON, *flags, "--swiglu", "--init_from_full_ckpt", path, "--ckpt_dir", str(tmp_path / "c")])
    new = consolidate_files(str(tmp_path / "c" / "epoch_1"))
    assert set(new) == set(sd)
    for k in sd:
        assert torch.equal(new[k].reshape(sd[k].shape), sd[k]), k  # lr 0: loaded verbatim
    out = _cli([*COMMON, *flags, "--init_from_full_ckpt", path, "--ckpt_dir", str(tmp_path / "d")], ok=False)
    assert "pass --swiglu to load it" in out


def test_full_checkpoint_refusals():
    def sd(**kw):
        return full_params_of(FSDPViT(tiny_cfg(**kw), dtype=torch.float32, seed=1))

    def load(sd_, **kw):
        FSDPViT(tiny_cfg(**kw), dtype=torch.float32, seed=2).load_full_state_dict(sd_)

    glu, gelu = sd(swiglu=True), sd()
    with pytest.raises(ValueError, match=r"uses --swiglu, but the checkpoint's MLP is not SwiGLU.*drop --swiglu"):
        load(gelu, swiglu=True)
    with pytest.raises(ValueError, match=r"the checkpoint's MLP is SwiGLU .*: pass --swiglu to load it"):
        load(glu)
    load(glu, swiglu=True)
    load(gelu)


def test_full_checkpoint_refusal_through_the_cli(tmp_path):
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    cfg = tiny_cfg(image_size=28, patch_size=14, embed_dim=32, num_heads=2, num_blocks=1, mlp_ratio=2.0)
    path = str(tmp_path / "gelu.pth")
    torch.save({"model": PlainViT(cfg).state_dict()}, path)
    out = _cli([*COMMON, "--mlp_ratio", "2", "--swiglu", "--init_from_full_ckpt", path,
                "--ckpt_dir", str(tmp_path / "c")], ok=False)
    assert "drop --swiglu to load it" in out


# ------------------------------------------------------------------------------------------------
# build: the new kernels compile for sm_90a without spills or serialised wgmma, the existing ones are unchanged
# ------------------------------------------------------------------------------------------------
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
GOLDEN = os.path.join(ROOT, "tests", "golden", "sass_before_swiglu.json")


def _symbol_key(name):
    """A kernel symbol without its anonymous-namespace tag: nvcc derives `_GLOBAL__N__<hash>_<len><file>_<hash>` from
    the source file's path, so the same kernel has another mangled name in every checkout."""
    return re.sub(r"_GLOBAL__N__[0-9a-f]+_(\d+)(\w*?)_[0-9a-f]{8}", r"_GLOBAL__N__\1\2", name)


def _sass_hash(obj, name):
    import hashlib

    out = subprocess.run(["cuobjdump", "-sass", "-fun", name, obj], capture_output=True, text=True, check=True).stdout
    ins = [re.sub(r"/\*[0-9a-f]{4,}\*/", "", ln).strip() for ln in out.splitlines() if ";" in ln]
    return hashlib.sha256("\n".join(ins).encode()).hexdigest()


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
@pytest.mark.parametrize("src,new", [("gemm_sm90.cu", ("gemm_glu_sm90_kernel",)),
                                     ("elementwise.cu", ("swiglu_fwd_kernel", "swiglu_bwd_kernel"))])
def test_kernels_compile_for_sm90a_without_spills_and_leave_existing_sass_unchanged(tmp_path, src, new):
    from vit_10b_fsdp_example_b200 import build_ext

    obj = str(tmp_path / "k.o")
    res = subprocess.run([NVCC, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, src), "-o", obj], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    log = res.stdout + res.stderr
    assert "C7510" not in log, "a call in a wgmma kernel serialises its MMAs"
    lines = log.splitlines()
    found = {}
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and any(n in ln for n in new):
            found[ln.split("'")[1]] = next(x for x in lines[i + 1:] if "spill stores" in x)
    # GEMM: {forward, dgrad} x block_n {128, 256} x cluster {1, 2}
    assert len(found) == (8 if src == "gemm_sm90.cu" else 2), list(found)
    assert all("0 bytes spill stores, 0 bytes spill loads" in v for v in found.values()), found
    if shutil.which("cuobjdump") is None:
        return
    for name in found:  # the new kernels make no calls (some pre-existing elementwise kernels do)
        fsass = subprocess.run(["cuobjdump", "-sass", "-fun", name, obj], capture_output=True, text=True).stdout
        assert "EXIT" in fsass and " CALL" not in fsass, name
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    golden = json.load(open(GOLDEN))
    ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != golden["nvcc"]:
        pytest.skip(f"the recorded SASS is from {golden['nvcc']}, this is {ver}")
    names = {_symbol_key(n): n for n in re.findall(r"Function : (\S+)", sass)}
    for key, h in golden["objects"][src].items():
        assert key in names, f"pre-existing kernel {key} is gone"
        assert _sass_hash(obj, names[key]) == h, f"SASS of pre-existing kernel {key} changed"
