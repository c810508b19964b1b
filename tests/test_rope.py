"""Rotary position embedding (--rope): the tables and the torch_ops reference against the closed form in float64, the
backward as the transpose, the relative-position property, the RoPE-fused QK norm against fp64 autograd, the engine
against an fp64 autograd oracle (q / k bias gradient included), FSDP equivalence, consolidation into PlainViT, the
flags and checkpoint records, the unchanged behaviour without the flag, and the build of the sm_90a kernels.

The closed form: hd = 4F; patch n of a g x g grid sits at t_r = (n // g) g_ref / g, t_c = (n % g) g_ref / g; pair i
(elements 2i, 2i + 1 of a head) turns by t_r theta^(-i / F) for i < F and by t_c theta^(-(i - F) / F) otherwise,
y0 = x0 cos - x1 sin, y1 = x1 cos + x0 sin.  Prefix tokens are not rotated; a kept patch turns by its own index."""
import json
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest
import torch
import torch.nn.functional as F

from dist_worker import launch
from helpers import full_grads_of, full_params_of, ptxas_usage, sass_hash, sass_symbol_key, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.models.plain import PlainViT
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW
from vit_10b_fsdp_example_b200.utils.checkpoint import load_ckpt, save_ckpt
from vit_10b_fsdp_example_b200.utils.schedule import get_warmup_cosine_scheduler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
IMAGES = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(7))
TARGET = torch.tensor([1, 5, 7, 2])
SITE_KEEP = 7_000_002


def angles64(grid, hd, theta=10000.0, ref_grid=0):
    """float64 [grid * grid, hd / 2]: the closed form, written independently of vit.rope_tables."""
    F_ = hd // 4
    g_ref = ref_grid or grid
    out = torch.empty(grid * grid, hd // 2, dtype=torch.float64)
    for n in range(grid * grid):
        t_r, t_c = (n // grid) * g_ref / grid, (n % grid) * g_ref / grid
        for i in range(hd // 2):
            out[n, i] = (t_r if i < F_ else t_c) * theta ** (-(i % F_) / F_)
    return out


def rotate64(x, ang, B, P, keep, H3):
    """float64 reference on [B * T, W] (W = H3 heads): rows of patch tokens turn by ang[table row]."""
    T = x.shape[0] // B
    y = x.double().clone()
    for b in range(B):
        for j in range(P, T):
            n = int(keep[b, j - P]) if keep is not None else j - P
            c, s = torch.cos(ang[n]), torch.sin(ang[n])
            row = y[b * T + j].view(H3, -1, 2)
            x0, x1 = row[..., 0].clone(), row[..., 1].clone()
            row[..., 0], row[..., 1] = x0 * c - x1 * s, x1 * c + x0 * s
    return y


def _keep(B, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randperm(N, generator=g)[:K].sort()[0] for _ in range(B)]).int()


# ------------------------------------------------------------------------------------------------
# tables and ops against the closed form
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid,hd,theta,ref", [(4, 8, 10000.0, 0), (5, 40, 10000.0, 0), (16, 160, 10000.0, 0),
                                               (7, 64, 100.0, 14), (3, 256, 10000.0, 2)])
def test_tables_are_the_closed_form_in_fp32(grid, hd, theta, ref):
    cos, sin = vit.rope_tables(grid, hd, theta, ref)
    ang = angles64(grid, hd, theta, ref)
    assert cos.dtype == sin.dtype == torch.float32 and cos.shape == (grid * grid, hd // 2)
    assert torch.equal(cos, torch.cos(ang).float()) and torch.equal(sin, torch.sin(ang).float())
    if ref in (0, grid):  # at the default the positions are the integer row and column
        rows = torch.arange(grid * grid).div(grid, rounding_mode="floor").double()
        assert torch.equal(cos[:, 0], torch.cos(rows).float())


@pytest.mark.parametrize("hd", [8, 40, 64, 160, 256])
@pytest.mark.parametrize("P", [0, 1, 5])
@pytest.mark.parametrize("with_keep", [False, True])
def test_rope_fwd_matches_fp64(hd, P, with_keep):
    grid, B, H = 3, 3, 2
    N = grid * grid
    K = 5 if with_keep else N  # T = P + K: 9 / 10 / 14 without keep, 5 / 6 / 10 with it
    keep = _keep(B, N, K, hd + P) if with_keep else None
    T = P + K
    cos, sin = vit.rope_tables(grid, hd, 10000.0)
    ang = angles64(grid, hd)
    g = torch.Generator().manual_seed(hd * 7 + P)
    x = torch.randn(B * T, 3 * H * hd, generator=g)
    want = rotate64(x[:, : 2 * H * hd], ang, B, P, keep, 2 * H)
    for inplace in (False, True):
        xi = x.clone()
        out = torch_ops.rope_fwd(xi, H, hd, cos, sin, B, P, keep, inplace=inplace)
        assert (out is xi) == inplace
        # fp32 rotation of fp32 inputs: the table error (half an ulp of cos / sin) times |x0| + |x1|, plus the rounding
        pairs = x[:, : 2 * H * hd].double().view(B * T, -1, 2).abs().sum(-1, keepdim=True).expand(-1, -1, 2)
        tol = 2 ** -23 * (2 * pairs + want.abs().view_as(pairs)).reshape(B * T, -1) + 1e-30
        assert ((out[:, : 2 * H * hd].double() - want).abs() <= tol).all()
        assert torch.equal(out[:, 2 * H * hd:], x[:, 2 * H * hd:])  # v
        pre = torch.cat([torch.arange(b * T, b * T + P) for b in range(B)])
        assert torch.equal(out[pre], x[pre])  # prefix rows, bit for bit
    xb = x.bfloat16()
    ob = torch_ops.rope_fwd(xb, H, hd, cos, sin, B, P, keep)
    wantb = rotate64(xb[:, : 2 * H * hd].float(), ang, B, P, keep, 2 * H)
    err = (ob[:, : 2 * H * hd].double() - wantb).abs()
    assert (err <= 2 ** -8 * wantb.abs() + 2 ** -22 * xb.float().abs().max().item() + 1e-30).all()  # one bf16 rounding
    assert torch.equal(ob[:, 2 * H * hd:], xb[:, 2 * H * hd:]) and torch.equal(ob[pre], xb[pre])


@pytest.mark.parametrize("hd,P,with_keep", [(8, 0, False), (40, 1, True), (160, 5, True), (64, 1, False)])
def test_backward_is_the_transpose_and_sums_the_returned_columns(hd, P, with_keep):
    grid, B, H = 4, 2, 3
    N = grid * grid
    K = 7 if with_keep else N
    keep = _keep(B, N, K, hd) if with_keep else None
    T = P + K
    cos, sin = vit.rope_tables(grid, hd, 10000.0)
    g = torch.Generator().manual_seed(hd)
    x = torch.randn(B * T, 3 * H * hd, generator=g)
    dy = torch.randn(B * T, 3 * H * hd, generator=g)
    rx = torch_ops.rope_fwd(x, H, hd, cos, sin, B, P, keep)
    rtg, cs = torch_ops.rope_bwd(dy.clone(), H, hd, cos, sin, B, P, keep)
    lhs = (rx.double() * dy.double()).sum().item()
    rhs = (x.double() * rtg.double()).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * (x.double().abs() * dy.double().abs()).sum().item()
    assert torch.equal(rtg[:, 2 * H * hd:], dy[:, 2 * H * hd:])  # dv untouched
    assert torch.allclose(cs.double(), rtg[:, : 2 * H * hd].double().sum(0), rtol=0, atol=1e-5)
    # R^T R = 1 on the rotated columns
    back, _ = torch_ops.rope_bwd(rx.clone(), H, hd, cos, sin, B, P, keep)
    assert torch.allclose(back, x, atol=1e-5)


def test_scores_depend_only_on_the_offset():
    """q(m) . k(n) after the rotation is a function of (r_m - r_n, c_m - c_n): the same q and k placed at two pairs
    of patches with the same offset give the same score."""
    grid, hd, H = 6, 32, 1
    N = grid * grid
    cos, sin = vit.rope_tables(grid, hd, 10000.0)
    g = torch.Generator().manual_seed(0)
    q, k = torch.randn(hd, generator=g), torch.randn(hd, generator=g)
    buf = torch.zeros(N, 3 * hd)
    buf[:, :hd] = q
    buf[:, hd: 2 * hd] = k
    r = torch_ops.rope_fwd(buf, H, hd, cos, sin, 1, 0).double()
    S = r[:, :hd] @ r[:, hd: 2 * hd].T  # S[m, n] = q(m) . k(n)
    seen = {}
    for m in range(N):
        for n in range(N):
            key = (m // grid - n // grid, m % grid - n % grid)
            seen.setdefault(key, []).append(S[m, n].item())
    for key, v in seen.items():
        assert max(v) - min(v) < 1e-4, (key, v)
    assert len({round(v[0], 3) for v in seen.values()}) > len(seen) // 2  # and the score does change with the offset


@pytest.mark.parametrize("hd,P,with_keep", [(8, 0, False), (40, 1, True), (64, 5, False), (160, 1, True)])
def test_fused_qk_norm_matches_fp64_autograd(hd, P, with_keep):
    grid, B, H = 3, 2, 2
    N = grid * grid
    K = 5 if with_keep else N
    keep = _keep(B, N, K, hd) if with_keep else None
    T = P + K
    D = H * hd
    cos, sin = vit.rope_tables(grid, hd, 10000.0)
    ang = angles64(grid, hd)
    g = torch.Generator().manual_seed(hd + P)
    qkv = torch.randn(B * T, 3 * D, generator=g) * 2 + 0.5
    wq, bq, wk, bk = (1 + 0.3 * torch.randn(hd, generator=g), 0.3 * torch.randn(hd, generator=g),
                      1 + 0.3 * torch.randn(hd, generator=g), 0.3 * torch.randn(hd, generator=g))
    dy = torch.randn(B * T, 3 * D, generator=g)
    rope = (cos, sin, B, P, keep)
    out, mean, rstd = torch_ops.qk_norm_fwd(qkv, H, hd, wq, bq, wk, bk, 1e-5, rope=rope)
    dq, dwq, dbq, dwk, dbk, cs = torch_ops.qk_norm_bwd(dy.clone(), qkv, H, hd, wq, wk, mean, rstd, rope=rope)

    p = [t.double().requires_grad_(True) for t in (qkv, wq, bq, wk, bk)]
    x = p[0][:, : 2 * D].reshape(B * T, 2, H, hd)
    y = torch.stack([F.layer_norm(x[:, 0], (hd,), p[1], p[2], 1e-5), F.layer_norm(x[:, 1], (hd,), p[3], p[4], 1e-5)], 1)
    y = y.reshape(B * T, 2 * D)
    # the rotation as a differentiable fp64 function
    idx = keep.long() if keep is not None else torch.arange(K).expand(B, K)
    c, s = torch.cos(ang)[idx][:, :, None], torch.sin(ang)[idx][:, :, None]
    yp = y.view(B, T, 2 * H, hd // 2, 2)
    x0, x1 = yp[:, P:, ..., 0], yp[:, P:, ..., 1]
    rot = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), -1)
    ref = torch.cat([yp[:, :P], rot], 1).reshape(B * T, 2 * D)
    ref.backward(dy[:, : 2 * D].double())
    assert torch.allclose(out[:, : 2 * D].double(), ref.detach(), atol=2e-5)
    assert torch.equal(out[:, 2 * D:], qkv[:, 2 * D:])
    assert torch.allclose(dq[:, : 2 * D].double(), p[0].grad[:, : 2 * D], atol=5e-5)
    for got, want in ((dwq, p[1].grad), (dbq, p[2].grad), (dwk, p[3].grad), (dbk, p[4].grad)):
        assert torch.allclose(got.double(), want, atol=1e-4)
    assert torch.allclose(cs.double(), p[0].grad[:, : 2 * D].sum(0), atol=1e-4)


def test_fused_reference_rounds_once():
    """bf16: the fused reference is the fp32 LayerNorm and rotation rounded once, not two rounded ops in a row."""
    grid, B, H, hd, P = 4, 2, 2, 64, 1
    T = P + grid * grid
    cos, sin = vit.rope_tables(grid, hd, 10000.0)
    g = torch.Generator().manual_seed(3)
    qkv = (torch.randn(B * T, 3 * H * hd, generator=g) * 3).bfloat16()
    w = [torch.ones(hd).bfloat16(), torch.zeros(hd).bfloat16()] * 2
    fused = torch_ops.qk_norm_fwd(qkv, H, hd, *w, 1e-5, rope=(cos, sin, B, P, None))[0]
    f32 = torch_ops.qk_norm_fwd(qkv.float(), H, hd, *[t.float() for t in w], 1e-5, rope=(cos, sin, B, P, None))[0]
    assert torch.equal(fused, f32.bfloat16())
    composed = torch_ops.rope_fwd(torch_ops.qk_norm_fwd(qkv, H, hd, *w, 1e-5)[0], H, hd, cos, sin, B, P)
    assert not torch.equal(fused, composed)


# ------------------------------------------------------------------------------------------------
# the engine against an fp64 autograd oracle
# ------------------------------------------------------------------------------------------------
def oracle_loss(cfg, params, images, target, keep=None, att_masks=None):
    """timm-style ViT with Eva's rotary embedding on q / k of the patch tokens (after the QK norm), optional prefix
    tokens, patch dropout pinned to keep [B, K] and attention-dropout factors per block [B, H, T, T]."""
    B = images.shape[0]
    D, H, hd, ps, P = cfg.embed_dim, cfg.num_heads, cfg.head_dim, cfg.patch_size, cfg.num_prefix_tokens
    w = params["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(D, 3, ps, ps)
    x = F.conv2d(images, w, params["patch_embed.proj.bias"], stride=ps).flatten(2).transpose(1, 2)
    pos = params["pos_embed"].view(1, cfg.pos_len, D)
    if cfg.class_token:
        prefix = [params["cls_token"].view(1, 1, D).expand(B, -1, -1)]
        if cfg.reg_tokens:
            prefix.append(params["reg_token"].view(1, -1, D).expand(B, -1, -1))
        x = torch.cat(prefix + [x], dim=1) + pos
    else:
        x = x + pos
    N = cfg.num_patches
    idx = keep.long() if keep is not None else torch.arange(N).expand(B, N)
    x = torch.cat([x[:, :P], x[:, P:].gather(1, idx[:, :, None].expand(-1, -1, D))], dim=1)
    T = x.shape[1]
    ang = angles64(cfg.grid, hd, cfg.rope_theta, cfg.rope_ref_grid)
    c, s = torch.cos(ang)[idx][:, None], torch.sin(ang)[idx][:, None]  # [B, 1, K, hd / 2]

    def rot(t):  # [B, H, T, hd]
        tp = t[:, :, P:].unflatten(-1, (-1, 2))
        t0, t1 = tp[..., 0], tp[..., 1]
        return torch.cat([t[:, :, :P], torch.stack((t0 * c - t1 * s, t1 * c + t0 * s), -1).flatten(-2)], dim=2)

    for i in range(cfg.num_blocks):
        g = lambda n: params[f"blocks.{i}.{n}"]  # noqa: E731
        h = F.layer_norm(x, (D,), g("norm1.weight"), g("norm1.bias"), 1e-5)
        q, k, v = F.linear(h, g("attn.qkv.weight"), g("attn.qkv.bias")).reshape(B, T, 3, H, hd).permute(2, 0, 3, 1, 4)
        if cfg.qk_norm:
            q = F.layer_norm(q, (hd,), g("attn.q_norm.weight"), g("attn.q_norm.bias"), 1e-5)
            k = F.layer_norm(k, (hd,), g("attn.k_norm.weight"), g("attn.k_norm.bias"), 1e-5)
        q, k = rot(q), rot(k)
        att = ((q @ k.transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1)
        if att_masks is not None:
            att = att * att_masks[i]
        a = (att @ v).transpose(1, 2).reshape(B, T, D)
        x = x + F.linear(a, g("attn.proj.weight"), g("attn.proj.bias"))
        h = F.layer_norm(x, (D,), g("norm2.weight"), g("norm2.bias"), 1e-5)
        x = x + F.linear(F.gelu(F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias"))), g("mlp.fc2.weight"),
                         g("mlp.fc2.bias"))
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x[:, 0] if cfg.class_token else x.mean(dim=1), params["head.weight"], params["head.bias"])
    return F.cross_entropy(logits, target)


def randomize(model, seed=0):
    """Prefix tokens, pos_embed and the QK-norm parameters at magnitudes that move the loss."""
    g = torch.Generator().manual_seed(seed)
    full = full_params_of(model)
    for k, v in full.items():
        if k in ("cls_token", "reg_token", "pos_embed"):
            full[k] = torch.randn(v.shape, generator=g)
        elif ".q_norm." in k or ".k_norm." in k:
            full[k] = (1.0 if k.endswith("weight") else 0.0) + 0.5 * torch.randn(v.shape, generator=g)
        elif k.endswith("attn.qkv.weight"):
            full[k] = v * 4  # larger scores: the rotation moves the softmax visibly
    model.load_full_state_dict(full)


def check_engine(model, images=IMAGES, target=TARGET):
    cfg, B = model.cfg, images.shape[0]
    model.drop.step = model.step_count
    keep = None
    if cfg.patch_drop_rate > 0:
        keep = torch.from_numpy(torch_ops.patch_drop_keep(model.drop.key(SITE_KEEP), B, cfg.num_patches, cfg.num_keep,
                                                          model.rank * B))
    att = None
    if cfg.att_dropout > 0:
        T, H = cfg.train_tokens, cfg.num_heads
        att = [torch_ops.dropout(torch.ones(B * H, T, T, dtype=torch.float64), cfg.att_dropout,
                                 model.drop.key(i * 8)).view(B, H, T, T) for i in range(cfg.num_blocks)]
    loss = model.forward_backward(images, target)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    ref = oracle_loss(cfg, params, images.double(), target, keep, att)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5, (loss.item(), ref.item())
    for name, p in params.items():
        gr = p.grad if p.grad is not None else torch.zeros_like(p)
        err = (got[name].double() - gr.view(got[name].shape)).abs().max().item()
        scale = gr.abs().max().item() + 1e-8
        assert err / scale < 2e-4, f"{name}: err {err} scale {scale}"
    return loss.item()


MODES = [dict(grad_ckpt=True, ckpt_keep_blocks=0), dict(grad_ckpt=True, ckpt_keep_blocks=99),
         dict(grad_ckpt=True, ckpt_keep_blocks=99, extras=True), dict(grad_ckpt=False)]
VARIANTS = [dict(), dict(class_token=True, reg_tokens=4), dict(patch_drop_rate=0.5),
            dict(class_token=True, reg_tokens=1, patch_drop_rate=0.5), dict(att_dropout=0.2),
            dict(rope_theta=100.0, rope_ref_grid=7)]


@pytest.mark.parametrize("qk_norm", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("mode", MODES)
def test_engine_matches_autograd(qk_norm, variant, mode):
    mode = dict(mode)
    extras = mode.pop("extras", False)
    model = FSDPViT(tiny_cfg(rope=True, qk_norm=qk_norm, **variant), dtype=torch.float32, seed=3, **mode)
    if extras:
        model.keep_extras = {"P": 99, "h": 99, "g": 99}
    randomize(model)
    check_engine(model)


def test_rope_changes_the_loss_and_the_qkv_bias_gradient():
    """The q / k bias gradient is the column sum after R^T: without rope_bwd's sums it would be those of the rotated
    gradient, which the oracle above would catch; here the two differ visibly."""
    a = FSDPViT(tiny_cfg(rope=True), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    randomize(a), randomize(b)
    assert abs(a.forward_backward(IMAGES, TARGET).item() - b.forward_backward(IMAGES, TARGET).item()) > 1e-4
    ga, gb = full_grads_of(a), full_grads_of(b)
    D = a.cfg.embed_dim
    assert (ga["blocks.0.attn.qkv.bias"][: 2 * D] - gb["blocks.0.attn.qkv.bias"][: 2 * D]).abs().max() > 1e-4


def test_eval_uses_the_full_grid():
    model = FSDPViT(tiny_cfg(rope=True, patch_drop_rate=0.5, class_token=True), dtype=torch.float32, seed=3)
    randomize(model)
    params = {k: v.double() for k, v in full_params_of(model).items()}
    with torch.no_grad():
        got = model.eval()(IMAGES)
    cfg = model.cfg
    # the oracle's loss with a one-hot target is -log_softmax[target]; compare through the loss of every class
    for t in range(3):
        tgt = torch.full((4,), t)
        want = oracle_loss(cfg, params, IMAGES.double(), tgt)
        assert abs(F.cross_entropy(got.double(), tgt).item() - want.item()) < 1e-5


# ------------------------------------------------------------------------------------------------
# FSDP equivalence, consolidation, checkpoints
# ------------------------------------------------------------------------------------------------
def test_two_ranks_reproduce_one(tmp_path):
    model = {"rope": True, "class_token": True, "reg_tokens": 1, "patch_drop_rate": 0.5}
    one = launch(1, {"model": model, "steps": 3}, str(tmp_path / "one.json"))
    two = launch(2, {"model": model, "steps": 3}, str(tmp_path / "two.json"))
    for a, b in zip(two["losses"], one["losses"]):
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b))
    for a, b in zip(two["norms"], one["norms"]):
        assert abs(a - b) <= 1e-4 * max(1.0, abs(b))


@pytest.mark.parametrize("kw", [dict(), dict(qk_norm=True, class_token=True, reg_tokens=2)])
def test_consolidated_checkpoint_loads_into_plain_vit(tmp_path, kw):
    d = str(tmp_path)
    prefix = os.path.join(d, "epoch_1")
    model = dict(rope=True, **kw)
    launch(2, {"model": model, "steps": 2, "seed": 7, "dump_state": prefix + "_rank_{rank}.ckpt"},
           os.path.join(d, "r.json"))
    full = consolidate_files(prefix, save_path=prefix + "_full.pth")
    cfg = tiny_cfg(**model)
    engine = FSDPViT(cfg, dtype=torch.float32, seed=99)
    engine.load_full_state_dict(full)
    plain = PlainViT.from_consolidated(prefix + "_full.pth", cfg).eval()
    assert set(plain.state_dict()) == set(full)  # the tables are not parameters
    images = torch.randn(3, 3, cfg.image_size, cfg.image_size)
    with torch.no_grad():
        want = plain(images)
    got = engine.eval()(images)
    assert torch.allclose(got, want, atol=1e-4), (got - want).abs().max()
    without = PlainViT.from_consolidated(prefix + "_full.pth", tiny_cfg(**kw)).eval()
    with torch.no_grad():
        assert not torch.allclose(without(images), want, atol=1e-4)


def test_plain_vit_with_a_pinned_subset_matches_the_engine():
    cfg = tiny_cfg(rope=True, class_token=True, reg_tokens=2, patch_drop_rate=0.5)
    engine = FSDPViT(cfg, dtype=torch.float32, seed=3)
    randomize(engine)
    engine.drop.step = engine.step_count
    keep = torch.from_numpy(torch_ops.patch_drop_keep(engine.drop.key(SITE_KEEP), 4, cfg.num_patches, cfg.num_keep, 0))
    loss = engine.forward_backward(IMAGES, TARGET)
    plain = PlainViT(cfg)
    sd = full_params_of(engine)
    sd["pos_embed"] = sd["pos_embed"][None]
    sd["cls_token"], sd["reg_token"] = sd["cls_token"][None], sd["reg_token"][None]
    sd["patch_embed.proj.weight"] = sd["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(cfg.embed_dim, 3, 8, 8)
    plain.load_state_dict(sd, strict=True)
    plain.train()
    want = F.cross_entropy(plain(IMAGES, patch_keep=keep), TARGET)
    assert abs(loss.item() - want.item()) < 1e-5


def _ckpt_roundtrip(tmp_path, save_cfg, load_cfg):
    m = FSDPViT(save_cfg, dtype=torch.float32, seed=1)
    opt = ShardedAdamW(m, lr=1e-3)
    sched = get_warmup_cosine_scheduler(opt, warmup_iteration=1, max_iteration=10)
    path = str(tmp_path / "e_rank_0.ckpt")
    save_ckpt(path, m, opt, sched, master_only=False)
    m2 = FSDPViT(load_cfg, dtype=torch.float32, seed=2)
    opt2 = ShardedAdamW(m2, lr=1e-3)
    load_ckpt(path, m2, opt2, get_warmup_cosine_scheduler(opt2, warmup_iteration=1, max_iteration=10))
    return torch.load(path, weights_only=False)


def test_checkpoints_record_the_settings_and_resume_refuses_others(tmp_path):
    on = tiny_cfg(rope=True, rope_theta=100.0, rope_ref_grid=8)
    ck = _ckpt_roundtrip(tmp_path, on, on)
    assert ck["rope"] == {"rope": True, "rope_theta": 100.0, "rope_ref_grid": 8}
    assert "rope" not in _ckpt_roundtrip(tmp_path, tiny_cfg(), tiny_cfg())  # no record: no RoPE
    with pytest.raises(ValueError, match=r"pass --rope --rope_theta 100 --rope_ref_grid 8 to resume"):
        _ckpt_roundtrip(tmp_path, on, tiny_cfg())
    with pytest.raises(ValueError, match="drop --rope, --rope_theta and --rope_ref_grid to resume"):
        _ckpt_roundtrip(tmp_path, tiny_cfg(), on)
    with pytest.raises(ValueError, match=r"pass --rope --rope_theta 100 --rope_ref_grid 8 to resume"):
        _ckpt_roundtrip(tmp_path, on, tiny_cfg(rope=True))


# ------------------------------------------------------------------------------------------------
# flags and config
# ------------------------------------------------------------------------------------------------
def test_cli_parsing_and_refusals(capsys):
    a = parse_args([])
    assert (a.rope, a.rope_theta, a.rope_ref_grid) == (False, 10000.0, 0)
    c = ViTConfig.from_args(parse_args(["--rope", "--rope_theta", "100", "--rope_ref_grid", "16"]))
    assert (c.rope, c.rope_theta, c.rope_ref_grid) == (True, 100.0, 16)
    for argv, msg in ((["--rope_theta", "100"], "--rope_theta needs --rope"),
                      (["--rope_ref_grid", "16"], "--rope_ref_grid needs --rope"),
                      (["--rope", "--embed_dim", "60", "--num_heads", "2"], "--rope needs head_dim % 4 == 0"),
                      (["--rope", "--rope_theta", "0"], "--rope_theta must be a finite number > 0"),
                      (["--rope", "--rope_theta", "inf"], "--rope_theta must be a finite number > 0"),
                      (["--rope", "--rope_theta", "nan"], "--rope_theta must be a finite number > 0"),
                      (["--rope", "--rope_ref_grid", "-1"], "--rope_ref_grid must be an integer >= 0")):
        with pytest.raises(SystemExit):
            parse_args(argv)
        assert msg in capsys.readouterr().err, argv
    parse_args(["--rope", "--embed_dim", "64", "--num_heads", "2"])
    with pytest.raises(ValueError, match="head_dim % 4 == 0"):
        tiny_cfg(rope=True, embed_dim=72, num_heads=4)  # hd 18
    with pytest.raises(ValueError, match="--rope_theta needs --rope"):
        tiny_cfg(rope_theta=5.0)
    with pytest.raises(ValueError, match="--rope_ref_grid needs --rope"):
        tiny_cfg(rope_ref_grid=4)
    with pytest.raises(ValueError, match="rope_theta must be a finite number > 0"):
        tiny_cfg(rope=True, rope_theta=-1.0)
    with pytest.raises(ValueError, match="rope_ref_grid must be an integer >= 0"):
        tiny_cfg(rope=True, rope_ref_grid=-2)
    assert tiny_cfg(rope=True).block_numel() == tiny_cfg().block_numel()  # no parameters


# ------------------------------------------------------------------------------------------------
# nothing new without the flag
# ------------------------------------------------------------------------------------------------
def _op_sequences():
    """The torch_ops calls (name and keyword names) of one training step and one eval per case, as recorded for
    tests/golden/ops_sequence_before_rope.json from the build before --rope existed."""
    cases = {
        "plain_ckpt": (dict(), dict(grad_ckpt=True, ckpt_keep_blocks=0)),
        "plain_kept": (dict(), dict(grad_ckpt=True, ckpt_keep_blocks=99)),
        "qk_norm_nockpt": (dict(qk_norm=True), dict(grad_ckpt=False)),
        "prefix_patch_drop_qk": (dict(qk_norm=True, class_token=True, reg_tokens=2, patch_drop_rate=0.5,
                                      att_dropout=0.1), dict(grad_ckpt=True, ckpt_keep_blocks=1)),
    }
    calls = []
    saved = {}
    names = [n for n in dir(torch_ops) if callable(getattr(torch_ops, n)) and not n.startswith("_")
             and getattr(getattr(torch_ops, n), "__module__", "") == torch_ops.__name__]
    for n in names:
        f = saved[n] = getattr(torch_ops, n)

        def wrap(*a, _f=f, _n=n, **k):
            calls.append(_n + ("(" + ",".join(sorted(k)) + ")" if k else ""))
            return _f(*a, **k)
        setattr(torch_ops, n, wrap)
    try:
        out = {}
        for name, (cfg, mode) in cases.items():
            calls.clear()
            m = FSDPViT(tiny_cfg(**cfg), dtype=torch.float32, seed=3, **mode)
            m.forward_backward(IMAGES, TARGET)
            m.eval()(IMAGES)
            out[name] = list(calls)
        return out
    finally:
        for n, f in saved.items():
            setattr(torch_ops, n, f)


def test_without_the_flag_the_op_sequence_is_the_one_before_rope():
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "ops_sequence_before_rope.json")))
    got = _op_sequences()
    assert got == want
    assert not any("rope" in c for seq in got.values() for c in seq)


def test_without_the_flag_no_rope_op_runs(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("rope op called without --rope")

    monkeypatch.setattr(torch_ops, "rope_fwd", boom)
    monkeypatch.setattr(torch_ops, "rope_bwd", boom)
    for kw in (dict(), dict(qk_norm=True), dict(class_token=True, patch_drop_rate=0.5)):
        for mode in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
            m = FSDPViT(tiny_cfg(**kw), dtype=torch.float32, seed=3, **mode)
            m.forward_backward(IMAGES, TARGET)
            m.eval()(IMAGES)
            assert m._rope_tables == {}


# ------------------------------------------------------------------------------------------------
# build: the new kernels, and every kernel recorded before --rope keeps its SASS
# ------------------------------------------------------------------------------------------------
def _compile(src, out_dir):
    from vit_10b_fsdp_example_b200 import build_ext

    obj = os.path.join(out_dir, src + ".o")
    res = subprocess.run([NVCC, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, src), "-o", obj], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    return obj, res.stdout + res.stderr


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("cuobjdump") is None, reason="needs nvcc and cuobjdump")
def test_rope_kernels_have_no_spills_or_calls(tmp_path):
    for src, pattern, count in (("rope.cu", "rope_kernel", 2), ("qk_norm.cu", "qk_norm_rope_", 7)):
        obj, log = _compile(src, str(tmp_path))
        usage = {k: v for k, v in ptxas_usage(log).items() if pattern in k}
        assert len(usage) == count, usage
        assert all(v[1] == v[2] == 0 for v in usage.values()), usage
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
        assert " CALL" not in sass


@pytest.mark.skipif(not os.path.exists(NVCC) or shutil.which("cuobjdump") is None, reason="needs nvcc and cuobjdump")
def test_every_kernel_recorded_before_rope_keeps_its_sass(tmp_path):
    """tests/golden/sass_before_rope.json holds every kernel of every object of the build before --rope; each keeps its
    SASS, registers and spills (new kernels may be added next to them)."""
    from vit_10b_fsdp_example_b200 import build_ext

    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_before_rope.json")))
    ver = subprocess.run([NVCC, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != golden["nvcc"]:
        pytest.skip(f"the recorded SASS is from {golden['nvcc']}, this is {ver}")
    srcs = sorted(golden["objects"])
    assert set(srcs) <= set(build_ext.CU_SOURCES)
    with ThreadPoolExecutor(len(srcs)) as ex:
        built = dict(zip(srcs, ex.map(lambda s: _compile(s, str(tmp_path)), srcs)))
    for src, (obj, log) in built.items():
        usage = ptxas_usage(log)
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
        names = {sass_symbol_key(n): n for n in re.findall(r"Function : (\S+)", sass)}
        missing = sorted(set(golden["objects"][src]) - set(names))
        assert not missing, f"{src}: kernels gone: {missing}"
        for key, want in golden["ptxas"][src].items():
            assert usage[key] == want, f"{src}: {key}: registers / spills {usage[key]}, were {want}"
        with ThreadPoolExecutor(8) as ex:
            hashes = dict(zip(golden["objects"][src], ex.map(lambda k: sass_hash(obj, names[k]),
                                                              golden["objects"][src])))
        changed = [k for k, h in golden["objects"][src].items() if hashes[k] != h]
        assert not changed, f"{src}: SASS of {len(changed)} kernels changed: {changed}"
