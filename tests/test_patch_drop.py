"""Patch dropout (--patch_drop_rate): the kept-patch selection (its count, order, reproducibility across world sizes and
steps, and its frequencies), the torch_ops reference of the gathered im2col, pos_gather and patch_drop_bwd against
fp64, the engine against an fp64 autograd oracle in timm's form, the behaviour at rate 0 and in eval, the keep-policy
byte counts, FSDP equivalence, resume, the CLI and the build of the sm_90a kernels.

The oracle follows timm's VisionTransformer.forward_features with PatchDropout(ordered=True): patch embed, + pos_embed
and the prefix tokens, pos_drop, then the gather of the kept patches (pinned to the reference selection), the blocks on
T' = P + K tokens, and the class-token or mean-pool head.  The pos-dropout mask is defined on the compacted buffer, so
the oracle applies it after the gather."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy import stats

from dist_worker import launch
from helpers import full_grads_of, full_params_of, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.models.plain import PlainViT
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT
from vit_10b_fsdp_example_b200.parallel.graph import GraphedTrainStep

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SITE = 7_000_002
IMAGES = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(7))
TARGET = torch.tensor([1, 5, 7, 2])


def pd_cfg(**kw):
    return tiny_cfg(**dict(dict(patch_drop_rate=0.5), **kw))


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


def next_keep(model, B):
    """The [B, K] kept patches the model's next training step draws (the reference selection)."""
    model.drop.step = model.step_count
    return torch.from_numpy(torch_ops.patch_drop_keep(model.drop.key(SITE), B, model.cfg.num_patches,
                                                      model.cfg.num_keep, model.rank * B))


# ------------------------------------------------------------------------------------------------
# selection
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid,R,K", [(2, 0.5, 2), (7, 0.25, 36), (14, 0.5, 98), (16, 0.5, 128), (16, 0.75, 64),
                                      (16, 0.999, 1), (37, 0.1, 1232), (7, 0.9, 4)])
def test_keep_count_is_timms(grid, R, K):
    N = grid * grid
    cfg = ViTConfig(image_size=14 * grid, patch_size=14, patch_drop_rate=R)
    assert cfg.num_keep == max(1, int(N * (1.0 - R))) == K
    assert cfg.train_tokens == K and cfg.num_tokens == N
    assert ViTConfig(image_size=14 * grid, class_token=True, reg_tokens=4, patch_drop_rate=R).train_tokens == 5 + K
    assert ViTConfig().num_keep == 256 and ViTConfig(class_token=True).train_tokens == 257


@pytest.mark.parametrize("B,N,K,offset", [(3, 16, 8, 0), (5, 49, 1, 7), (4, 196, 196, 3), (2, 1369, 684, 100)])
def test_selection_is_ascending_unique_and_inverse_is_consistent(B, N, K, offset):
    keep, inv = torch_ops.patch_drop_select(1234 + N, B, N, K, offset, "cpu")
    assert keep.dtype == torch.int32 and inv.dtype == torch.int32 and keep.shape == (B, K) and inv.shape == (B, N)
    k = keep.long()
    assert (k >= 0).all() and (k < N).all()
    assert (k[:, 1:] > k[:, :-1]).all()  # strictly ascending, so unique
    assert ((inv >= 0).sum(1) == K).all() and ((inv >= -1) & (inv < K)).all()
    for b in range(B):
        assert torch.equal(inv[b, k[b]], torch.arange(K, dtype=torch.int32))


def test_selection_is_the_k_smallest_philox_draws():
    key, B, N, K, off = 987654321, 3, 50, 20, 11
    keep = torch_ops.patch_drop_keep(key, B, N, K, off)
    for b in range(B):
        r = [int(torch_ops.philox4x32_10([n // 4], [off + b], key & 0xFFFFFFFF, key >> 32)[n % 4][0]) for n in range(N)]
        want = sorted(sorted(range(N), key=lambda n: (r[n], n))[:K])
        assert keep[b].tolist() == want


def test_same_subset_at_every_world_size_and_a_new_one_next_step():
    ctx = vit.DropoutCtx(seed=3)
    full = torch_ops.patch_drop_keep(ctx.key(SITE), 8, 64, 32, 0)
    for W in (1, 2, 4):
        local = 8 // W
        parts = [torch_ops.patch_drop_keep(ctx.key(SITE), local, 64, 32, r * local) for r in range(W)]
        assert np.array_equal(np.concatenate(parts), full)
    ctx.step += 1
    nxt = torch_ops.patch_drop_keep(ctx.key(SITE), 8, 64, 32, 0)
    assert not np.array_equal(nxt, full)
    assert len({tuple(row) for row in full}) == 8  # every image its own subset


@pytest.mark.parametrize("N,K", [(49, 24), (196, 98), (16, 3)])
def test_every_patch_is_kept_with_frequency_k_over_n(N, K):
    """Over 20000 images the per-patch keep counts follow Binomial(B, K / N): the chi-square statistic (with the
    binomial variance) is consistent with N - 1 degrees of freedom (the counts sum to B * K)."""
    B = 20000
    keep = torch_ops.patch_drop_keep(vit.DropoutCtx(seed=N).key(SITE), B, N, K, 0)
    counts = np.bincount(keep.ravel(), minlength=N)
    p = K / N
    stat = float((((counts - B * p) ** 2) / (B * p * (1 - p))).sum())
    assert stats.chi2.sf(stat, N - 1) > 1e-4, stat
    assert np.abs(counts / B - p).max() < 6 * math.sqrt(p * (1 - p) / B)


# ------------------------------------------------------------------------------------------------
# ops against fp64
# ------------------------------------------------------------------------------------------------
MIXES = [None, (0.3, None), (0.6, (2, 19, 5, 30))]


@pytest.mark.parametrize("mix", MIXES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gathered_im2col_against_fp64(mix, dtype):
    B, S, P, kpad = 4, 32, 8, 200
    images = torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(1))
    keep, _ = torch_ops.patch_drop_select(55, B, 16, 6, 2, "cpu")
    cols = torch_ops.patch_im2col(images, P, kpad, dtype, mix=mix, keep=keep)
    assert cols.shape == (B * 6, kpad) and cols.dtype == dtype
    full = torch_ops.patch_im2col(images, P, kpad, dtype, mix=mix)
    rows = (torch.arange(B)[:, None] * 16 + keep.long()).reshape(-1)
    assert torch.equal(cols, full[rows])  # exactly the kept rows of the full im2col
    x = images.double()
    mag = torch.zeros_like(x)  # Mixup in fp32: two products and a sum, each rounded once
    if mix is not None:
        lam, box = mix
        if box is None:
            mag = 2.0 ** -23 * (x.abs() * lam + x.flip(0).abs() * (1 - lam))
            x = x * lam + x.flip(0) * (1 - lam)
        else:
            x = x.clone()
            x[:, :, box[0]:box[1], box[2]:box[3]] = images.double().flip(0)[:, :, box[0]:box[1], box[2]:box[3]]

    def kept(t):
        t = t.view(B, 3, 4, P, 4, P).permute(0, 2, 4, 1, 3, 5).reshape(B, 16, 3 * P * P)
        return torch.gather(t, 1, keep.long()[:, :, None].expand(-1, -1, 3 * P * P)).reshape(-1, 3 * P * P)

    want = kept(x)
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -24
    assert ((cols[:, : 3 * P * P].double() - want).abs() <= ulp * want.abs() + kept(mag) * (1 + ulp) + 1e-30).all()
    assert (cols[:, 3 * P * P:] == 0).all()


def test_pos_gather_and_patch_drop_bwd_against_fp64():
    g = torch.Generator().manual_seed(3)
    B, N, K, D = 5, 12, 7, 16
    pos = torch.randn(N, D, generator=g).bfloat16()
    keep, inv = torch_ops.patch_drop_select(77, B, N, K, 4, "cpu")
    assert torch.equal(torch_ops.pos_gather(pos, keep).view(B, K, D), pos[keep.long()])
    for P in (0, 1, 3):
        dx0 = torch.randn(B * (P + K), D, generator=g).bfloat16()
        dpatch, dtok = torch_ops.patch_drop_bwd(dx0, inv, B, N, K, P)
        x = dx0.double().view(B, P + K, D)
        if P:
            assert torch.equal(dpatch, dx0.view(B, P + K, D)[:, P:].reshape(B * K, D))
        else:
            assert dpatch is None
        want = torch.zeros(P + N, D, dtype=torch.float64)
        mag = torch.zeros(P + N, D, dtype=torch.float64)
        want[:P] = x[:, :P].sum(0)
        mag[:P] = x[:, :P].abs().sum(0)
        for b in range(B):
            want[P + keep[b].long()] += x[b, P:]
            mag[P + keep[b].long()] += x[b, P:].abs()
        assert dtok.dtype == torch.float32 and dtok.shape == (P + N, D)
        # at most B fp32 additions per entry: error <= B * 2^-24 * sum |terms|
        assert ((dtok.double() - want).abs() <= B * 2.0 ** -24 * mag).all()
        dropped = (inv == -1).all(0)
        assert (dtok[P:][dropped] == 0).all()


# ------------------------------------------------------------------------------------------------
# the engine against the fp64 oracle
# ------------------------------------------------------------------------------------------------
def oracle_loss(cfg, params, images, target, keep, masks=None, pos_mask=None, soft=None):
    """timm VisionTransformer(patch_drop_rate=R) in training with the subset `keep` [B, K] pinned; optional QK norm,
    LayerScale, SwiGLU, dropout / drop-path factors (per block {"att", "proj", "fc1", "fc2", "sa", "sm"}), a
    pos-dropout factor on the compacted [B, T', D] buffer and soft targets."""
    B = images.shape[0]
    D, H, hd, ps, P = cfg.embed_dim, cfg.num_heads, cfg.head_dim, cfg.patch_size, cfg.num_prefix_tokens
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
    x = torch.cat([x[:, :P], x[:, P:].gather(1, keep.long()[:, :, None].expand(-1, -1, D))], dim=1)  # PatchDropout
    if pos_mask is not None:
        x = x * pos_mask
    T = x.shape[1]
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
        u = F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias"))
        if cfg.swiglu:
            gate, val = u.chunk(2, dim=-1)
            h = m("fc1", F.silu(gate) * val)
        else:
            h = m("fc1", F.gelu(u))
        x = x + ls("ls2.gamma", m("sm", m("fc2", F.linear(h, g("mlp.fc2.weight"), g("mlp.fc2.bias")))))
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x[:, 0] if cfg.class_token else x.mean(dim=1), params["head.weight"], params["head.bias"])
    if soft is not None:
        return (-soft.double() * torch.log_softmax(logits, dim=-1)).sum(-1).mean()
    return F.cross_entropy(logits, target)


def _check_against_oracle(model, images, target, **kw):
    keep = next_keep(model, images.shape[0])
    loss = model.forward_backward(images, target)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    ref_loss = oracle_loss(model.cfg, params, kw.pop("oracle_images", images).double(), target, keep, **kw)
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
    return keep


VARIANTS = [dict(), dict(class_token=True), dict(class_token=True, reg_tokens=4),
            dict(class_token=True, no_embed_class=True)]
MODES = [dict(grad_ckpt=True, ckpt_keep_blocks=0), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=99),
         dict(grad_ckpt=True, ckpt_keep_blocks=1, flatten_parameters=True)]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", MODES)
def test_engine_matches_autograd(variant, mode):
    model = FSDPViT(pd_cfg(**variant), dtype=torch.float32, seed=3, **mode)
    if mode.get("ckpt_keep_blocks") == 99:
        model.keep_extras = {"P": 99, "h": 99, "g": 99}
    randomize(model)
    images = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(1))
    keep = _check_against_oracle(model, images, TARGET)
    assert keep.shape == (4, 8)
    assert len({tuple(r) for r in keep.tolist()}) > 1  # the images keep different patches


@pytest.mark.parametrize("R", [0.25, 0.75, 0.95])
def test_other_rates_and_the_flash_style_path(monkeypatch, R):
    monkeypatch.setattr(torch_ops, "FLASH_ATTENTION", True)
    for variant in (dict(), dict(class_token=True, reg_tokens=2)):
        model = FSDPViT(pd_cfg(patch_drop_rate=R, **variant), dtype=torch.float32, seed=3, ckpt_keep_blocks=1)
        randomize(model, seed=2)
        _check_against_oracle(model, IMAGES, TARGET)


def _model_masks(model, B):
    """The dropout / drop-path factors the model's next training step draws, on T' tokens per image."""
    cfg, ctx = model.cfg, model.drop
    ctx.step = model.step_count
    T, H, D = cfg.train_tokens, cfg.num_heads, cfg.embed_dim
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
            m["fc1"] = torch_ops.dropout(torch.ones(B * T, cfg.mlp_out_dim, dtype=torch.float64), pm,
                                         ctx.key(site + 2)).view(B, T, -1)
            m["fc2"] = torch_ops.dropout(torch.ones(B * T, D, dtype=torch.float64), pm, ctx.key(site + 3)).view(B, T, D)
        if rate > 0:
            for name, off in (("sa", 4), ("sm", 5)):
                m[name] = torch_ops.drop_path_scale(ctx.key(site + off), rate, B, model.rank * B,
                                                    "cpu").double().view(B, 1, 1)
        out.append(m)
    pos_mask = None
    if cfg.pos_dropout > 0:  # on the compacted buffer
        pos_mask = torch_ops.dropout(torch.ones(B * T, D, dtype=torch.float64), cfg.pos_dropout,
                                     ctx.key(7_000_001)).view(B, T, D)
    return out, pos_mask


@pytest.mark.parametrize("kw", [dict(qk_norm=True, init_values=1e-5), dict(swiglu=True),
                                dict(swiglu=True, class_token=True, mlp_dropout=0.2),
                                dict(att_dropout=0.2, pos_dropout=0.3),
                                dict(drop_path_rate=0.5, init_values=1e-5, qk_norm=True, class_token=True),
                                dict(att_dropout=0.1, mlp_dropout=0.1, pos_dropout=0.1, drop_path_rate=0.5,
                                     class_token=True, reg_tokens=2, no_embed_class=True)])
@pytest.mark.parametrize("mode", [dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)])
def test_composes_with_other_features(kw, mode):
    cfg = pd_cfg(num_blocks=4, **kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3, **mode)
    randomize(model, seed=3)
    images = torch.randn(8, 3, 32, 32, generator=torch.Generator().manual_seed(2))
    target = torch.randint(0, 10, (8,), generator=torch.Generator().manual_seed(2))
    masks, pos_mask = _model_masks(model, 8)
    _check_against_oracle(model, images, target, masks=masks, pos_mask=pos_mask)


@pytest.mark.parametrize("kw", [dict(mixup=0.8, smoothing=0.1), dict(cutmix=1.0, smoothing=0.1, class_token=True)])
def test_mixup_and_cutmix_mix_before_the_selection(kw):
    cfg = pd_cfg(**kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3)
    randomize(model, seed=4)
    mix = vit.draw_mix(cfg, vit.mix_rng(model.drop.seed, model.step_count, model.rank))
    assert mix is not None
    soft = torch_ops.mixup_target(TARGET, cfg.num_classes, mix[0], cfg.smoothing)
    _check_against_oracle(model, IMAGES, TARGET, oracle_images=torch_ops.mix_images(IMAGES, mix), soft=soft)


# ------------------------------------------------------------------------------------------------
# eval, rate 0, byte counts, FSDP, resume
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
def test_eval_uses_every_patch_and_equals_the_rate_0_model(variant):
    a = FSDPViT(pd_cfg(**variant), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(**variant), dtype=torch.float32, seed=3)
    randomize(a)
    randomize(b)
    for k, v in full_params_of(a).items():
        assert torch.equal(v, full_params_of(b)[k])
    assert torch.equal(a.eval()(IMAGES), b.eval()(IMAGES))
    plain = PlainViT(a.cfg).eval()
    plain.load_state_dict({k: v.view(plain.state_dict()[k].shape) for k, v in full_params_of(a).items()})
    with torch.no_grad():
        assert torch.allclose(plain(IMAGES), a.eval()(IMAGES), atol=1e-5)


@pytest.mark.parametrize("variant", [dict(), dict(class_token=True, reg_tokens=2)])
def test_plain_vit_patch_dropout_with_a_pinned_subset_matches_the_engine(variant):
    model = FSDPViT(pd_cfg(**variant), dtype=torch.float32, seed=3)
    randomize(model)
    keep = next_keep(model, 4)
    loss = model.forward_backward(IMAGES, TARGET)
    plain = PlainViT(model.cfg).train()
    plain.load_state_dict({k: v.view(plain.state_dict()[k].shape) for k, v in full_params_of(model).items()})
    with torch.no_grad():
        ref = F.cross_entropy(plain(IMAGES, patch_keep=keep), TARGET)
        assert abs(ref.item() - loss.item()) < 1e-5
        free = plain(IMAGES)  # timm's own random subset: a different, valid draw
        assert free.shape == (4, 10) and torch.isfinite(free).all()


def test_rate_0_calls_nothing_new(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("patch-dropout op called at patch_drop_rate 0")

    for name in ("patch_drop_select", "pos_gather", "patch_drop_bwd"):
        monkeypatch.setattr(torch_ops, name, boom)
    im2col = torch_ops.patch_im2col

    def no_keep(*a, **k):
        assert "keep" not in k
        return im2col(*a, **k)

    monkeypatch.setattr(torch_ops, "patch_im2col", no_keep)
    for variant in (dict(), dict(class_token=True)):
        for kw in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
            model = FSDPViT(tiny_cfg(drop_path_rate=0.3, pos_dropout=0.1, **variant), dtype=torch.float32, seed=3,
                            **kw)
            model.forward_backward(IMAGES, TARGET)
            model.eval()(IMAGES)
    # and in eval with the flag on
    model = FSDPViT(pd_cfg(), dtype=torch.float32, seed=3)
    model.eval()(IMAGES)
    assert [n for n, _ in vit.root_param_specs(pd_cfg())] == [n for n, _ in vit.root_param_specs(tiny_cfg())]
    assert pd_cfg().total_numel() == tiny_cfg().total_numel()


def test_lean_and_extra_bytes_use_the_training_token_count():
    for variant in (dict(), dict(class_token=True, reg_tokens=4)):
        a = FSDPViT(pd_cfg(qk_norm=True, **variant), dtype=torch.float32, seed=3)
        b = FSDPViT(tiny_cfg(qk_norm=True, **variant), dtype=torch.float32, seed=3)
        T, Tp = b.cfg.num_tokens, a.cfg.train_tokens
        assert Tp == a.cfg.num_prefix_tokens + 8 and Tp < T
        assert a.lean_bytes_per_block(4) * T == b.lean_bytes_per_block(4) * Tp
        eb = dict(a.extra_bytes_per_block(4))
        assert eb["h"] == 2 * 4 * Tp * a.cfg.embed_dim * 4
        assert eb["P"] == 4 * a.cfg.num_heads * Tp * ((Tp + 7) // 8 * 8) * 4
        assert eb["g"] == 4 * Tp * a.cfg.mlp_out_dim * 4


def test_gradients_of_one_step_equal_across_checkpoint_modes():
    grads = []
    for mode in MODES:
        model = FSDPViT(pd_cfg(class_token=True, reg_tokens=2), dtype=torch.float32, seed=3, **mode)
        randomize(model)
        model.forward_backward(IMAGES, TARGET)
        grads.append(full_grads_of(model))
    for g in grads[1:]:
        for k, v in g.items():
            assert torch.allclose(v, grads[0][k], atol=1e-6, rtol=1e-5), k


MODEL = dict(patch_drop_rate=0.5, class_token=True, reg_tokens=1)


@pytest.fixture(scope="module")
def pd_baseline(tmp_path_factory):
    out = tmp_path_factory.mktemp("pd_base") / "r.json"
    return launch(1, {"model": MODEL, "steps": 4}, str(out))


def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.mark.parametrize("opts", [{}, {"no_fsdp": True}])
def test_two_ranks_reproduce_one(opts, pd_baseline, tmp_path):
    res = launch(2, dict(opts, model=MODEL, steps=4), str(tmp_path / "r.json"))
    _close(res["losses"], pd_baseline["losses"])
    _close(res["norms"], pd_baseline["norms"], tol=1e-4)


def test_resume_equals_uninterrupted(tmp_path):
    d = str(tmp_path)
    model = dict(patch_drop_rate=0.25)
    full = launch(2, {"model": model, "steps": 5}, os.path.join(d, "full.json"))
    launch(2, {"model": model, "steps": 3, "save_at": 3, "save_path": os.path.join(d, "e1_rank_{rank}.ckpt")},
           os.path.join(d, "part.json"))
    rest = launch(2, {"model": model, "steps": 5, "resume_from": os.path.join(d, "e1_rank_{rank}.ckpt"),
                      "resume_step": 3}, os.path.join(d, "rest.json"))
    for a, b in zip(rest["losses"], full["losses"][3:]):
        assert abs(a - b) < 1e-6


# ------------------------------------------------------------------------------------------------
# CLI, config, CUDA graphs, build
# ------------------------------------------------------------------------------------------------
def test_cli_parsing_and_rejections(capsys):
    assert parse_args([]).patch_drop_rate == 0.0
    args = parse_args(["--patch_drop_rate", "0.5", "--class_token"])
    cfg = ViTConfig.from_args(args)
    assert cfg.patch_drop_rate == 0.5 and cfg.num_keep == 128 and cfg.train_tokens == 129
    for bad in ("1.0", "-0.1", "1.5", "nan"):
        with pytest.raises(SystemExit):
            parse_args(["--patch_drop_rate", bad])
        assert "--patch_drop_rate must be in [0, 1)" in capsys.readouterr().err
    for bad in (1.0, -0.5):
        with pytest.raises(ValueError, match="patch_drop_rate must be in"):
            ViTConfig(patch_drop_rate=bad)


def test_cuda_graph_training_refuses_patch_dropout():
    model = FSDPViT(pd_cfg(), dtype=torch.float32, seed=3)
    with pytest.raises(RuntimeError, match="patch_drop_rate > 0"):
        GraphedTrainStep(model, None)
    model.eval()
    with pytest.raises(RuntimeError, match="CUDA graphs need a CUDA model"):  # eval passes the patch-dropout check
        GraphedTrainStep(model, None)


NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")


@pytest.mark.skipif(not os.path.exists(NVCC), reason="needs nvcc")
def test_kernels_compile_for_sm90a_without_spills_or_calls(tmp_path):
    from vit_10b_fsdp_example_b200 import build_ext

    obj = str(tmp_path / "pd.o")
    res = subprocess.run([NVCC, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, "patch_drop.cu"), "-o", obj], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    spills = [ln for ln in res.stderr.splitlines() if "spill" in ln]
    assert len(spills) == 9 and all("0 bytes spill stores, 0 bytes spill loads" in ln for ln in spills), spills
    if shutil.which("cuobjdump") is None:
        return
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    for kernel in ("patch_drop_select_kernel", "im2col_gather_kernel", "pos_gather_kernel", "patch_drop_bwd_kernel"):
        assert kernel in sass, kernel
    assert " CALL" not in sass and "EXIT" in sass
