"""Class and register tokens (--class_token / --reg_tokens / --no_embed_class): the torch_ops reference of the token
assembly and its backward against fp64, the engine against an fp64 autograd oracle written in timm's form, parameters,
the CLI, FSDP equivalence, checkpoints (timm-layout state dicts and the refusals) and the build of the sm_90a kernels.

The oracle follows timm's VisionTransformer literally: x = cat(cls, reg, patches) + pos (or cat(prefix, patches + pos)
with no_embed_class), pos_drop, the blocks on all T tokens, norm(x)[:, 0], head.  The prefix tokens start at 1e-6 in a
real run, so every engine check here randomises them (and pos_embed) to make a wrong gradient visible."""
import math
import os
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


def pt_cfg(**kw):
    return tiny_cfg(**dict(dict(class_token=True), **kw))


def randomize(model, seed=0):
    """Prefix tokens, pos_embed and the LayerScale / QK-norm parameters at magnitudes that move the loss."""
    g = torch.Generator().manual_seed(seed)
    full = full_params_of(model)
    for k, v in full.items():
        if k in ("cls_token", "reg_token", "pos_embed"):
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
@pytest.mark.parametrize("P", [1, 2, 5])
@pytest.mark.parametrize("embed", [True, False])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ops_against_fp64(P, embed, dtype):
    B, N, D = 3, 9, 16
    g = torch.Generator().manual_seed(P * 10 + embed)
    y = torch.randn(B * N, D, generator=g).to(dtype)
    cls = torch.randn(1, D, generator=g).to(dtype)
    reg = torch.randn(P - 1, D, generator=g).to(dtype) if P > 1 else None
    pos = torch.randn(P, D, generator=g).to(dtype) if embed else None
    x0 = torch_ops.tokens_fwd(y, cls, reg, pos, B, N)
    assert x0.shape == (B * (N + P), D) and x0.dtype == dtype
    pre = torch.cat([cls.double()] + ([reg.double()] if reg is not None else []))
    if embed:
        pre = pre + pos.double()
    want = torch.cat([pre[None].expand(B, P, D), y.double().view(B, N, D)], dim=1).reshape(-1, D)
    x = x0.double().view(B, N + P, D)
    assert torch.equal(x[:, P:], y.double().view(B, N, D))  # the patch rows are copied
    # the prefix rows: one fp32 sum rounded once to the dtype -> within half an ulp of the exact sum
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -23
    assert ((x0.double() - want).abs() <= ulp * want.abs() + 1e-30).all()

    dx0 = torch.randn(B * (N + P), D, generator=g).to(dtype)
    dpatch, dtok = torch_ops.tokens_bwd(dx0, B, N, P)
    assert dpatch.shape == (B * N, D) and dpatch.is_contiguous() and dtok.dtype == torch.float32
    assert torch.equal(dpatch, dx0.view(B, N + P, D)[:, P:].reshape(B * N, D))
    want_tok = dx0.double().view(B, N + P, D).sum(0)
    # B fp32 additions: error <= B * 2^-24 * sum |dx0|
    bound = B * 2.0 ** -24 * dx0.double().abs().view(B, N + P, D).sum(0)
    assert ((dtok.double() - want_tok).abs() <= bound).all()

    # and against autograd on timm's form
    c, r, p_, yy = (t.double().requires_grad_(True) if t is not None else None for t in (cls, reg, pos, y))
    prefix = torch.cat([c[None].expand(B, 1, D)] + ([r[None].expand(B, P - 1, D)] if r is not None else []), dim=1)
    xx = torch.cat([prefix, yy.view(B, N, D)], dim=1)
    if embed:
        xx = xx + torch.cat([p_, torch.zeros(N, D, dtype=torch.float64)])[None]
    xx.reshape(-1, D).backward(dx0.double())
    assert torch.allclose(dtok[0].double(), c.grad[0], rtol=1e-5, atol=1e-6)
    if r is not None:
        assert torch.allclose(dtok[1:P].double(), r.grad, rtol=1e-5, atol=1e-6)
    if embed:
        assert torch.allclose(dtok[:P].double(), p_.grad, rtol=1e-5, atol=1e-6)
    assert torch.equal(dpatch.double(), yy.grad)


# ------------------------------------------------------------------------------------------------
# the engine against the fp64 oracle
# ------------------------------------------------------------------------------------------------
def autograd_vit_loss_timm(cfg, params, images, target, masks=None, pos_mask=None, soft=None):
    """timm VisionTransformer(class_token=True, reg_tokens=R, no_embed_class=...) with the optional QK norm, LayerScale,
    dropout / drop-path factors (masks: per-block dict {"att", "proj", "fc1", "fc2", "sa", "sm"}), a pos-dropout factor
    [B, T, D] and soft targets (Mixup / smoothing)."""
    B = images.shape[0]
    N, T, D, H, hd, ps = cfg.num_patches, cfg.num_tokens, cfg.embed_dim, cfg.num_heads, cfg.head_dim, cfg.patch_size
    w = params["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(D, 3, ps, ps)
    x = F.conv2d(images, w, params["patch_embed.proj.bias"], stride=ps).flatten(2).transpose(1, 2)
    prefix = [params["cls_token"].view(1, 1, D).expand(B, -1, -1)]
    if cfg.reg_tokens:
        prefix.append(params["reg_token"].view(1, -1, D).expand(B, -1, -1))
    pos = params["pos_embed"].view(1, cfg.pos_len, D)
    if cfg.no_embed_class:
        x = torch.cat(prefix + [x + pos], dim=1)
    else:
        x = torch.cat(prefix + [x], dim=1) + pos
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
        h = m("fc1", F.gelu(F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias"))))
        x = x + ls("ls2.gamma", m("sm", m("fc2", F.linear(h, g("mlp.fc2.weight"), g("mlp.fc2.bias")))))
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x[:, 0], params["head.weight"], params["head.bias"])
    if soft is not None:
        return (-soft.double() * torch.log_softmax(logits, dim=-1)).sum(-1).mean(), logits
    return F.cross_entropy(logits, target), logits


def _check_against_oracle(model, images, target, **kw):
    loss = model.forward_backward(images, target)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    assert params["cls_token"].abs().max() > 0.1  # randomised, not the 1e-6 start
    ref_loss, ref_logits = autograd_vit_loss_timm(model.cfg, params, images.double(), target, **kw)
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


VARIANTS = [dict(), dict(reg_tokens=4), dict(no_embed_class=True), dict(reg_tokens=2, no_embed_class=True)]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("grad_ckpt,keep,flatten", [(True, 0, False), (False, 0, False), (True, 0, True),
                                                    (True, 1, False), (True, 99, True)])
def test_engine_matches_autograd(variant, grad_ckpt, keep, flatten):
    cfg = pt_cfg(**variant)
    model = FSDPViT(cfg, dtype=torch.float32, grad_ckpt=grad_ckpt, ckpt_keep_blocks=keep, flatten_parameters=flatten,
                    seed=3)
    randomize(model)
    images = torch.randn(4, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(1))
    ref_logits = _check_against_oracle(model, images, TARGET)
    assert torch.allclose(model.eval()(images).double(), ref_logits.detach(), atol=1e-4)


@pytest.mark.parametrize("extras", [{"P": 99, "h": 99, "g": 99}, {"P": 1, "h": 0, "g": 1}])
def test_kept_blocks_with_extras_match_autograd(extras):
    model = FSDPViT(pt_cfg(reg_tokens=3), dtype=torch.float32, grad_ckpt=True, ckpt_keep_blocks=99, seed=3)
    model.keep_extras = extras
    randomize(model, seed=1)
    _check_against_oracle(model, IMAGES, TARGET)


@pytest.mark.parametrize("kw", [dict(), dict(qk_norm=True), dict(init_values=1e-5, qk_norm=True, reg_tokens=4)])
def test_flash_style_path_qk_norm_and_layer_scale_match_autograd(monkeypatch, kw):
    monkeypatch.setattr(torch_ops, "FLASH_ATTENTION", True)
    for mode in (dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)):
        model = FSDPViT(pt_cfg(**kw), dtype=torch.float32, seed=3, **mode)
        randomize(model, seed=2)
        _check_against_oracle(model, IMAGES, TARGET)


def _model_masks(model, B):
    """The multiplicative dropout / drop-path factors the model's blocks draw in its next training step, on T tokens."""
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
            m["fc1"] = torch_ops.dropout(torch.ones(B * T, cfg.hidden_dim, dtype=torch.float64), pm,
                                         ctx.key(site + 2)).view(B, T, -1)
            m["fc2"] = torch_ops.dropout(torch.ones(B * T, D, dtype=torch.float64), pm, ctx.key(site + 3)).view(B, T, D)
        if rate > 0:
            for name, off in (("sa", 4), ("sm", 5)):
                m[name] = torch_ops.drop_path_scale(ctx.key(site + off), rate, B, model.rank * B,
                                                    "cpu").double().view(B, 1, 1)
        out.append(m)
    pos_mask = None
    if cfg.pos_dropout > 0:  # applied to all T rows, like timm's pos_drop after the concatenation
        pos_mask = torch_ops.dropout(torch.ones(B * T, D, dtype=torch.float64), cfg.pos_dropout,
                                     ctx.key(7_000_001)).view(B, T, D)
    return out, pos_mask


@pytest.mark.parametrize("kw", [dict(att_dropout=0.2), dict(mlp_dropout=0.2), dict(pos_dropout=0.3),
                                dict(drop_path_rate=0.5, init_values=1e-5, qk_norm=True),
                                dict(att_dropout=0.1, mlp_dropout=0.1, pos_dropout=0.1, drop_path_rate=0.5,
                                     reg_tokens=2, no_embed_class=True)])
@pytest.mark.parametrize("mode", [dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)])
def test_composes_with_dropout_and_drop_path(kw, mode):
    cfg = pt_cfg(num_blocks=4, **kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3, **mode)
    randomize(model, seed=3)
    images = torch.randn(8, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(2))
    target = torch.randint(0, 10, (8,), generator=torch.Generator().manual_seed(2))
    masks, pos_mask = _model_masks(model, 8)
    _check_against_oracle(model, images, target, masks=masks, pos_mask=pos_mask)


@pytest.mark.parametrize("kw", [dict(mixup=0.8, smoothing=0.1), dict(cutmix=1.0, smoothing=0.1, reg_tokens=2)])
def test_mixup_and_smoothing_match_autograd(kw):
    cfg = pt_cfg(**kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3)
    randomize(model, seed=4)
    mix = vit.draw_mix(cfg, vit.mix_rng(model.drop.seed, model.step_count, model.rank))
    assert mix is not None
    mixed = torch_ops.mix_images(IMAGES, mix)
    soft = torch_ops.mixup_target(TARGET, cfg.num_classes, mix[0], cfg.smoothing)
    loss = model.forward_backward(IMAGES, TARGET)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    ref_loss, _ = autograd_vit_loss_timm(cfg, params, mixed.double(), TARGET, soft=soft)
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
        raise AssertionError("prefix-token op called without --class_token")

    monkeypatch.setattr(torch_ops, "tokens_fwd", boom)
    monkeypatch.setattr(torch_ops, "tokens_bwd", boom)
    for kw in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
        model = FSDPViT(tiny_cfg(drop_path_rate=0.3, pos_dropout=0.1), dtype=torch.float32, seed=3, **kw)
        model.forward_backward(IMAGES, TARGET)
        model.eval()(IMAGES)
    names = [n for n, _ in vit.root_param_specs(tiny_cfg())]
    assert names == ["patch_embed.proj.weight", "patch_embed.proj.bias", "pos_embed", "norm.weight", "norm.bias",
                     "head.weight", "head.bias"]


def test_parameters_order_shapes_and_counts():
    cfg = pt_cfg(reg_tokens=4)
    D, N = cfg.embed_dim, cfg.num_patches
    specs = dict(vit.root_param_specs(cfg))
    assert list(specs) == ["patch_embed.proj.weight", "patch_embed.proj.bias", "cls_token", "reg_token", "pos_embed",
                           "norm.weight", "norm.bias", "head.weight", "head.bias"]
    assert specs["cls_token"] == (1, D) and specs["reg_token"] == (4, D) and specs["pos_embed"] == (N + 5, D)
    assert vit.logical_shapes(cfg) == {"patch_embed.proj.weight": (D, 3, 8, 8), "pos_embed": (1, N + 5, D),
                                       "cls_token": (1, 1, D), "reg_token": (1, 4, D)}
    assert (cfg.num_prefix_tokens, cfg.num_tokens, cfg.pos_len) == (5, N + 5, N + 5)
    ne = pt_cfg(reg_tokens=4, no_embed_class=True)
    assert (ne.num_prefix_tokens, ne.num_tokens, ne.pos_len) == (5, N + 5, N)
    assert dict(vit.root_param_specs(ne))["pos_embed"] == (N, D)
    base = tiny_cfg()
    assert (base.num_prefix_tokens, base.num_tokens, base.pos_len) == (0, N, N)
    for c in (cfg, ne, base, pt_cfg()):
        assert c.root_numel() == sum(torch.Size(s).numel() for n, s in vit.root_param_specs(c)
                                     if n != "patch_embed.proj.weight") + D * c.patch_k
        assert c.block_numel() == base.block_numel()
    assert cfg.root_numel() == base.root_numel() + 2 * 5 * D
    assert ne.root_numel() == base.root_numel() + 5 * D
    assert ViTConfig(class_token=True).num_tokens == 257 and ViTConfig(class_token=True, reg_tokens=4).num_tokens == 261


def test_init_draws_after_every_existing_parameter():
    """--class_token --no_embed_class: every pre-existing parameter equals the same-seed model without the flags."""
    a = full_params_of(FSDPViT(pt_cfg(reg_tokens=3, no_embed_class=True), dtype=torch.float32, seed=5))
    b = full_params_of(FSDPViT(tiny_cfg(), dtype=torch.float32, seed=5))
    assert set(a) - set(b) == {"cls_token", "reg_token"}
    for k, v in b.items():
        assert torch.equal(a[k], v), k
    for k in ("cls_token", "reg_token"):  # normal(std=1e-6)
        assert a[k].abs().max() < 1e-5 and a[k].std() > 1e-7 and a[k].abs().max() > 0
    # embedded prefix: pos_embed is one [N + P, D] trunc-normal draw in its place, so the blocks are still the same
    c = full_params_of(FSDPViT(pt_cfg(reg_tokens=3), dtype=torch.float32, seed=5))
    assert c["pos_embed"].shape == (tiny_cfg().num_patches + 4, tiny_cfg().embed_dim)
    assert c["pos_embed"].std() == pytest.approx(0.02, rel=0.2)
    assert all(torch.equal(c[k], v) for k, v in b.items() if k.startswith("blocks.") or k.startswith("patch_embed."))


def test_lean_bytes_and_flops_count_every_token():
    a = FSDPViT(pt_cfg(reg_tokens=4), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    N, T = a.cfg.num_patches, a.cfg.num_tokens
    assert a.lean_bytes_per_block(4) * N == b.lean_bytes_per_block(4) * T
    qa = FSDPViT(pt_cfg(qk_norm=True), dtype=torch.float32, seed=3)
    qb = FSDPViT(tiny_cfg(qk_norm=True), dtype=torch.float32, seed=3)
    assert qa.lean_bytes_per_block(4) * N == qb.lean_bytes_per_block(4) * (N + 1)
    eb = dict(a.extra_bytes_per_block(4))
    assert eb["h"] == 2 * 4 * T * a.cfg.embed_dim * 4
    assert eb["P"] == 4 * a.cfg.num_heads * T * ((T + 7) // 8 * 8) * 4
    c, c0 = ViTConfig(class_token=True), ViTConfig()
    D, Hd, L = c.embed_dim, c.hidden_dim, c.num_blocks
    per_block = lambda n: 2 * n * (3 * D * D + D * D + 2 * D * Hd) + 4 * n * n * D  # noqa: E731
    assert c.flops_per_image() - c0.flops_per_image() == 4.0 * L * (per_block(257) - per_block(256))


def test_cli_parsing_and_rejections():
    args = parse_args([])
    assert (args.class_token, args.reg_tokens, args.no_embed_class) == (False, 0, False)
    c = ViTConfig.from_args(args)
    assert (c.class_token, c.reg_tokens, c.no_embed_class) == (False, 0, False)
    args = parse_args(["--class_token", "--reg_tokens", "4", "--no_embed_class"])
    c = ViTConfig.from_args(args)
    assert (c.class_token, c.reg_tokens, c.no_embed_class, c.num_prefix_tokens) == (True, 4, True, 5)
    for bad in (["--reg_tokens", "4"], ["--no_embed_class"], ["--class_token", "--reg_tokens", "-1"],
                ["--class_token", "--reg_tokens", "1.5"]):
        with pytest.raises(SystemExit):
            parse_args(bad)
    with pytest.raises(ValueError, match="--reg_tokens needs --class_token"):
        tiny_cfg(reg_tokens=2)
    with pytest.raises(ValueError, match="--no_embed_class needs --class_token"):
        tiny_cfg(no_embed_class=True)
    with pytest.raises(ValueError, match="reg_tokens must be an integer >= 0"):
        pt_cfg(reg_tokens=-1)


def test_cli_refusal_message(tmp_path):
    r = subprocess.run([sys.executable, "run_vit_training.py", "--reg_tokens", "4"], cwd=ROOT, capture_output=True,
                       text=True, timeout=120)
    assert r.returncode != 0 and "--reg_tokens needs --class_token" in r.stderr


# ------------------------------------------------------------------------------------------------
# FSDP equivalence and checkpoints
# ------------------------------------------------------------------------------------------------
MODEL = {"class_token": True, "reg_tokens": 2}


@pytest.fixture(scope="module")
def pt_baseline(tmp_path_factory):
    out = tmp_path_factory.mktemp("pt_base") / "r.json"
    return launch(1, {"model": MODEL, "steps": 4}, str(out))


def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.mark.parametrize("opts", [{}, {"flatten": True}])
def test_two_ranks_reproduce_one(opts, pt_baseline, tmp_path):
    res = launch(2, dict(opts, model=MODEL, steps=4), str(tmp_path / "r.json"))
    _close(res["losses"], pt_baseline["losses"])
    _close(res["norms"], pt_baseline["norms"], tol=1e-4)


def test_resume_equals_uninterrupted(tmp_path):
    d = str(tmp_path)
    model = dict(MODEL, no_embed_class=True)
    full = launch(2, {"model": model, "steps": 5}, os.path.join(d, "full.json"))
    launch(2, {"model": model, "steps": 3, "save_at": 3, "save_path": os.path.join(d, "e1_rank_{rank}.ckpt")},
           os.path.join(d, "part.json"))
    rest = launch(2, {"model": model, "steps": 5, "resume_from": os.path.join(d, "e1_rank_{rank}.ckpt"),
                      "resume_step": 3}, os.path.join(d, "rest.json"))
    for a, b in zip(rest["losses"], full["losses"][3:]):
        assert abs(a - b) < 1e-6


@pytest.mark.parametrize("no_embed_class", [False, True])
def test_consolidated_checkpoint_loads_into_plain_vit_and_back(tmp_path, no_embed_class):
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    d = str(tmp_path)
    prefix = os.path.join(d, "epoch_1")
    model = dict(MODEL, no_embed_class=no_embed_class)
    launch(2, {"model": model, "steps": 2, "seed": 7, "dump_state": prefix + "_rank_{rank}.ckpt"},
           os.path.join(d, "r.json"))
    full = consolidate_files(prefix, save_path=prefix + "_full.pth")
    cfg = pt_cfg(reg_tokens=2, no_embed_class=no_embed_class)
    D = cfg.embed_dim
    assert full["cls_token"].shape == (1, 1, D) and full["reg_token"].shape == (1, 2, D)
    assert full["pos_embed"].shape == (1, cfg.pos_len, D)
    images = torch.randn(3, 3, cfg.image_size, cfg.image_size)
    engine = FSDPViT(cfg, dtype=torch.float32, seed=99)
    engine.load_full_state_dict(full)
    plain = PlainViT.from_consolidated(prefix + "_full.pth", cfg).eval()
    assert set(plain.state_dict()) == set(full)
    with torch.no_grad():
        assert torch.allclose(engine.eval()(images), plain(images), atol=1e-4)
    # prefix tokens and pos_embed at magnitudes that matter, then engine -> PlainViT -> engine
    randomize(engine, seed=5)
    sd = full_params_of(engine)
    for k, shape in vit.logical_shapes(cfg).items():
        sd[k] = sd[k][:, : cfg.patch_k].reshape(shape) if k == "patch_embed.proj.weight" else sd[k].reshape(shape)
    plain.load_state_dict(sd, strict=True)
    with torch.no_grad():
        want = plain(images)
    got = engine.eval()(images)
    assert torch.allclose(got, want, atol=1e-4), (got - want).abs().max()
    back = FSDPViT(cfg, dtype=torch.float32, seed=5)
    back.load_full_state_dict(plain.state_dict())
    assert torch.allclose(back.eval()(images), want, atol=1e-4)


def _timm_resample(posemb, new_grid, num_prefix_tokens):
    """timm 0.4.12's resize_pos_embed (the timm version the blocks here follow), re-implemented: the first
    num_prefix_tokens rows are kept, the grid is resampled with F.interpolate(bicubic, align_corners=False).  (Later
    timm releases, resample_abs_pos_embed, default to antialias=True, which is another bicubic kernel even when
    growing the grid; this loader does not use it.)"""
    prefix, grid = posemb[:, :num_prefix_tokens], posemb[:, num_prefix_tokens:]
    g0 = int(math.sqrt(grid.shape[1]))
    D = grid.shape[2]
    grid = grid.reshape(1, g0, g0, D).permute(0, 3, 1, 2).float()
    grid = F.interpolate(grid, size=(new_grid, new_grid), mode="bicubic", align_corners=False)
    grid = grid.permute(0, 2, 3, 1).reshape(1, new_grid * new_grid, D)
    return torch.cat([prefix, grid], dim=1)


def _cli(args, ok=True):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "run_vit_training.py", *args], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=300)
    assert (r.returncode == 0) == ok, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout + r.stderr


COMMON = ["--fake_data", "--device", "cpu", "--nproc", "1", "--image_size", "42", "--patch_size", "14",
          "--embed_dim", "32", "--num_heads", "2", "--num_blocks", "1", "--num_classes", "10", "--batch_size", "4",
          "--warmup_steps", "1", "--max_steps", "1", "--num_workers", "0", "--num_epochs", "1",
          "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--lr", "0", "--weight_decay", "0"]


def test_timm_layout_state_dict_loads_with_prefix_rows_verbatim(tmp_path):
    """A timm-style checkpoint (cls_token, 2 reg_token, a wrapper prefix, pos_embed [1, 3 + 2x2, D]) starts a 3x3-grid
    run: the prefix tokens and the first 3 pos_embed rows arrive verbatim, the grid is resampled as timm does."""
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    D = 32
    src = PlainViT(tiny_cfg(image_size=28, patch_size=14, embed_dim=D, num_heads=2, num_blocks=1, mlp_ratio=4.0,
                            class_token=True, reg_tokens=2))
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(v.shape, generator=g) for k, v in src.state_dict().items()}
    assert sd["pos_embed"].shape == (1, 3 + 4, D)
    wrapped = {("module." + k if k == "cls_token" else k): v for k, v in sd.items()}
    path = str(tmp_path / "timm.pth")
    torch.save(wrapped, path)
    out = _cli([*COMMON, "--class_token", "--reg_tokens", "2", "--init_from_full_ckpt", path,
                "--ckpt_dir", str(tmp_path / "c")])
    assert "pos_embed resampled from 4 to 9 tokens" in out
    new = consolidate_files(str(tmp_path / "c" / "epoch_1"))
    assert torch.equal(new["cls_token"], sd["cls_token"]) and torch.equal(new["reg_token"], sd["reg_token"])
    assert new["pos_embed"].shape == (1, 3 + 9, D)
    assert torch.equal(new["pos_embed"][:, :3], sd["pos_embed"][:, :3])
    want = _timm_resample(sd["pos_embed"], 3, 3)
    assert torch.allclose(new["pos_embed"], want, rtol=0, atol=1e-6), (new["pos_embed"] - want).abs().max()
    assert torch.equal(new["blocks.0.attn.qkv.weight"], sd["blocks.0.attn.qkv.weight"])


def test_resize_pos_embed_with_prefix_rows():
    from vit_10b_fsdp_example_b200.utils.checkpoint import resize_pos_embed

    pe = torch.randn(1, 5 + 16, 8)
    out = resize_pos_embed(pe, 49, 8, num_prefix_tokens=5)
    assert out.shape == (1, 5 + 49, 8) and torch.equal(out[:, :5], pe[:, :5])
    assert torch.equal(out[:, 5:], resize_pos_embed(pe[:, 5:], 49, 8))
    assert resize_pos_embed(pe, 16, 8, num_prefix_tokens=5) is pe
    with pytest.raises(ValueError, match="cannot resample 20 to 49 tokens after its 1 prefix rows"):
        resize_pos_embed(pe, 49, 8, num_prefix_tokens=1)


def test_full_checkpoint_refusals():
    def sd(**kw):
        return full_params_of(FSDPViT(tiny_cfg(**kw), dtype=torch.float32, seed=1))

    def load(sd_, **kw):
        FSDPViT(tiny_cfg(**kw), dtype=torch.float32, seed=2).load_full_state_dict(sd_)

    cls, plain_ = sd(class_token=True), sd()
    with pytest.raises(ValueError, match=r"uses --class_token, but the checkpoint has no cls_token.*drop --class_"):
        load(plain_, class_token=True)
    with pytest.raises(ValueError, match="trained with a class token\\): pass --class_token"):
        load(cls)
    with pytest.raises(ValueError, match="has 4 register tokens \\(reg_token\\) and this model 0: pass --reg_tokens 4"):
        load(sd(class_token=True, reg_tokens=4), class_token=True)
    with pytest.raises(ValueError, match="has 0 register tokens \\(reg_token\\) and this model 2: drop --reg_tokens"):
        load(cls, class_token=True, reg_tokens=2)
    with pytest.raises(ValueError, match="prefix tokens were position-embedded, drop --no_embed_class"):
        load(cls, class_token=True, no_embed_class=True)
    with pytest.raises(ValueError, match="without the 1 prefix tokens: pass --no_embed_class"):
        load(sd(class_token=True, no_embed_class=True), class_token=True)
    bad = dict(cls, pos_embed=torch.zeros(7, tiny_cfg().embed_dim))
    with pytest.raises(ValueError, match="pos_embed has 7 rows, but this model needs 1 prefix rows plus a square grid"):
        load(bad, class_token=True)
    for kw in (dict(class_token=True), dict(class_token=True, reg_tokens=4, no_embed_class=True), dict()):
        load(sd(**kw), **kw)  # the matching pairs load


def test_full_checkpoint_refusal_through_the_cli(tmp_path):
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    cfg = tiny_cfg(image_size=42, patch_size=14, embed_dim=32, num_heads=2, num_blocks=1, mlp_ratio=4.0,
                   class_token=True)
    path = str(tmp_path / "cls.pth")
    torch.save({"model": PlainViT(cfg).state_dict()}, path)
    out = _cli([*COMMON, "--init_from_full_ckpt", path, "--ckpt_dir", str(tmp_path / "c")], ok=False)
    assert "pass --class_token to load it" in out
    out = _cli([*COMMON, "--class_token", "--no_embed_class", "--init_from_full_ckpt", path,
                "--ckpt_dir", str(tmp_path / "d")], ok=False)
    assert "drop --no_embed_class to load it" in out


# ------------------------------------------------------------------------------------------------
# build: the new kernels compile for sm_90a without spills or calls
# ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")),
                    reason="needs nvcc")
def test_prefix_token_kernels_compile_for_sm90a_without_spills(tmp_path):
    import shutil

    from vit_10b_fsdp_example_b200 import build_ext

    nvcc = os.path.join(build_ext._cuda_home(), "bin", "nvcc")
    res = subprocess.run([nvcc, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, "prefix_tokens.cu"), "-o", str(tmp_path / "p.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = (res.stdout + res.stderr).splitlines()
    found = {}
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln:
            assert "sm_90a" in ln
            found[ln.split("'")[1]] = next(x for x in lines[i + 1:] if "spill stores" in x)
    assert len(found) == 2 and {k for k in found if "tokens_fwd_kernel" in k or "tokens_bwd_kernel" in k} == set(found)
    assert all("0 bytes spill stores, 0 bytes spill loads" in v for v in found.values()), found
    if shutil.which("cuobjdump"):
        sass = subprocess.run(["cuobjdump", "-sass", str(tmp_path / "p.o")], capture_output=True, text=True).stdout
        assert "tokens_fwd_kernel" in sass and " CALL" not in sass
