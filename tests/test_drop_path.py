"""Stochastic depth (--drop_path_rate): timm drop_path semantics, masks, hand-written backward, FSDP equivalence, CLI.

The CPU path (torch_ops) draws the per-sample masks with a NumPy Philox-4x32-10 that reproduces csrc/dropout.cuh bit
for bit; the GPU tests (test_gpu_drop_path.py) hold the kernels to it."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dist_worker import launch
from helpers import full_grads_of, full_params_of, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

IMAGES = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(7))
TARGET = torch.tensor([1, 5, 7, 2])


# ------------------------------------------------------------------------------------------------
# rates and masks
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate,depth", [(0.0, 3), (0.1, 12), (0.3, 32), (0.5, 1), (0.2, 2)])
def test_rates_are_timm_linspace(rate, depth):
    cfg = tiny_cfg(drop_path_rate=rate, num_blocks=depth)
    assert vit.drop_path_rates(cfg) == [x.item() for x in torch.linspace(0, rate, depth)]
    assert vit.drop_path_rates(cfg)[0] == 0.0


def test_rate_zero_builds_no_masks_and_calls_no_new_op(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("drop-path op called at rate 0")

    monkeypatch.setattr(torch_ops, "drop_path_scale", boom)
    monkeypatch.setattr(torch_ops, "drop_path_bwd", boom)
    for kw in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
        FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3, **kw).forward_backward(IMAGES, TARGET)
    cfg = tiny_cfg()
    p = vit.init_block_params(cfg, torch.Generator().manual_seed(0))
    x = torch.randn(4 * cfg.num_patches, cfg.embed_dim)
    _, s = vit.block_forward(torch_ops, cfg, p, x, 4, save=True, drop=vit.DropoutCtx(1), block_idx=2)
    assert "dpath" not in s


def test_block_zero_takes_the_plain_path(monkeypatch):
    """Block 0 always has rate 0: it draws no masks even when the model's rate is > 0."""
    calls = []
    real = torch_ops.drop_path_scale
    monkeypatch.setattr(torch_ops, "drop_path_scale", lambda *a, **k: calls.append(a) or real(*a, **k))
    cfg = tiny_cfg(drop_path_rate=0.4)
    p = vit.init_block_params(cfg, torch.Generator().manual_seed(0))
    x = torch.randn(4 * cfg.num_patches, cfg.embed_dim)
    _, s = vit.block_forward(torch_ops, cfg, p, x, 4, save=True, drop=vit.DropoutCtx(1), block_idx=0)
    assert not calls and "dpath" not in s
    _, s = vit.block_forward(torch_ops, cfg, p, x, 4, save=True, drop=vit.DropoutCtx(1), block_idx=1)
    assert len(calls) == 2 and s["dpath"][0].shape == (4,)


def _philox_scalar(c0, c1, k0, k1):
    """Python-int transcription of philox4x32_10 in csrc/dropout.cuh (an independent check of the NumPy one)."""
    c2, c3 = 0x5EED5EED, 0x0B200B20
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & 0xFFFFFFFF, (p0 >> 32) ^ c3 ^ k1, p0 & 0xFFFFFFFF
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def test_numpy_philox_matches_scalar_transcription():
    rng = np.random.default_rng(0)
    c0 = rng.integers(0, 2 ** 32, 64, dtype=np.uint64)
    c1 = rng.integers(0, 2 ** 32, 64, dtype=np.uint64)
    for k0, k1 in ((0, 0), (0xDEADBEEF, 0x12345678), (0xFFFFFFFF, 0x7FFFFFFF)):
        got = torch_ops.philox4x32_10(c0, c1, k0, k1)
        for j in range(64):
            ref = _philox_scalar(int(c0[j]), int(c1[j]), k0, k1)
            assert tuple(int(g[j]) for g in got) == ref


def test_mask_definition_is_dropout_keep8():
    key, p, B, off = 0x0123_4567_89AB_CDEF, 0.3, 37, 13
    keep = torch_ops.drop_path_keep(key, p, B, off)
    t = torch_ops.dropout_thresh16(p)
    for b in range(B):
        g = off + b
        r = _philox_scalar(g // 8, 0, key & 0xFFFFFFFF, key >> 32)
        chunk = (r[(g % 8) >> 1] >> (16 * (g % 2))) & 0xFFFF
        assert bool(keep[b]) == (chunk >= t)


@pytest.mark.parametrize("p", [0.05, 0.1, 0.3, 0.5, 0.9])
def test_keep_fraction_matches_quantised_probability(p):
    n = 100_000
    keep = torch_ops.drop_path_keep(0xABCDEF12345, p, n, 0)
    q = 1.0 - torch_ops.dropout_thresh16(p) / 65536.0
    sigma = (q * (1 - q) / n) ** 0.5
    assert abs(keep.mean() - q) < 5 * sigma, (keep.mean(), q)
    s = torch_ops.drop_path_scale(0xABCDEF12345, p, 8, 0, "cpu")
    assert set(s.tolist()) <= {0.0, torch_ops.dropout_scale(torch_ops.dropout_thresh16(p))}
    assert torch_ops.dropout_scale(torch_ops.dropout_thresh16(p)) == pytest.approx(1.0 / q, rel=1e-6)


def test_keys_and_offsets_give_different_masks_same_key_same_mask():
    a = torch_ops.drop_path_keep(11, 0.5, 4096, 0)
    assert (a == torch_ops.drop_path_keep(11, 0.5, 4096, 0)).all()
    assert (a != torch_ops.drop_path_keep(12, 0.5, 4096, 0)).any()
    assert (a != torch_ops.drop_path_keep(11, 0.5, 4096, 8)).any()
    # the offset selects a window of one global stream: rank r's images are samples r * B_local + b
    assert (a[100:300] == torch_ops.drop_path_keep(11, 0.5, 200, 100)).all()
    ctx = vit.DropoutCtx(5)
    assert ctx.key(1 * 8 + 4) != ctx.key(1 * 8 + 5)


# ------------------------------------------------------------------------------------------------
# hand-written backward vs autograd
# ------------------------------------------------------------------------------------------------
def autograd_vit_loss_dp(cfg, params, images, target, scales):
    """timm-style ViT with drop_path as the per-sample scale vectors `scales[i] = (attention, mlp)` (None = block kept
    whole): x = x + s_att[b] * attn(norm1(x)); x = x + s_mlp[b] * mlp(norm2(x))."""
    B = images.shape[0]
    N, D, H, hd, P = cfg.num_patches, cfg.embed_dim, cfg.num_heads, cfg.head_dim, cfg.patch_size
    w = params["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(D, 3, P, P)
    x = F.conv2d(images, w, params["patch_embed.proj.bias"], stride=P).flatten(2).transpose(1, 2)
    x = x + params["pos_embed"].view(1, N, D)
    for i in range(cfg.num_blocks):
        g = lambda n: params[f"blocks.{i}.{n}"]  # noqa: E731
        s_att, s_mlp = (None, None) if scales[i] is None else (s.to(x.dtype).view(B, 1, 1) for s in scales[i])
        h = F.layer_norm(x, (D,), g("norm1.weight"), g("norm1.bias"), 1e-5)
        qkv = F.linear(h, g("attn.qkv.weight"), g("attn.qkv.bias")).reshape(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
        att = ((qkv[0] @ qkv[1].transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1)
        a = F.linear((att @ qkv[2]).transpose(1, 2).reshape(B, N, D), g("attn.proj.weight"), g("attn.proj.bias"))
        x = x + (a if s_att is None else a * s_att)
        h = F.layer_norm(x, (D,), g("norm2.weight"), g("norm2.bias"), 1e-5)
        m = F.gelu(F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias")))
        m = F.linear(m, g("mlp.fc2.weight"), g("mlp.fc2.bias"))
        x = x + (m if s_mlp is None else m * s_mlp)
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x.mean(dim=1), params["head.weight"], params["head.bias"])
    return F.cross_entropy(logits, target), logits


def model_scales(model, B):
    """The scale vectors the model's blocks draw in its next training step."""
    ctx, cfg = model.drop, model.cfg
    out = []
    for i, r in enumerate(vit.drop_path_rates(cfg)):
        if r == 0:
            out.append(None)
            continue
        key = vit.DropoutCtx.key(ctx, i * 8 + 4), vit.DropoutCtx.key(ctx, i * 8 + 5)
        out.append(tuple(torch_ops.drop_path_scale(k, r, B, model.rank * B, "cpu") for k in key))
    return out


@pytest.mark.parametrize("grad_ckpt,keep", [(True, 0), (False, 0), (True, 1), (True, 99)])
def test_grads_match_autograd(grad_ckpt, keep):
    torch.manual_seed(0)
    cfg = tiny_cfg(drop_path_rate=0.5, num_blocks=4)
    model = FSDPViT(cfg, dtype=torch.float32, grad_ckpt=grad_ckpt, ckpt_keep_blocks=keep, seed=3)
    images = torch.randn(8, 3, cfg.image_size, cfg.image_size)
    target = torch.randint(0, 10, (8,))
    scales = model_scales(model, 8)
    dropped = sum(int((s == 0).sum()) for sc in scales if sc is not None for s in sc)
    assert dropped > 0 and any(sc is not None and (sc[0] > 0).any() for sc in scales)  # both kinds of sample occur
    loss = model.forward_backward(images, target)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    ref_loss, _ = autograd_vit_loss_dp(cfg, params, images.double(), target, scales)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 1e-5
    for name, p in params.items():
        g = p.grad if p.grad is not None else torch.zeros_like(p)
        err = (got[name].double() - g).abs().max().item()
        scale = g.abs().max().item() + 1e-8
        assert err / scale < 2e-4, f"{name}: err {err} scale {scale}"


def test_with_mlp_dropout_recompute_and_kept_blocks_agree():
    cfg = tiny_cfg(drop_path_rate=0.5, mlp_dropout=0.1, att_dropout=0.1, pos_dropout=0.1)
    grads = []
    for ckpt, keep in ((True, 0), (False, 0), (True, 1), (True, 99)):
        model = FSDPViT(cfg, dtype=torch.float32, grad_ckpt=ckpt, ckpt_keep_blocks=keep, seed=3)
        model.forward_backward(IMAGES, TARGET)
        grads.append(full_grads_of(model))
    for other in grads[1:]:
        for k in grads[0]:
            assert torch.allclose(grads[0][k], other[k], atol=1e-6), k
    # and the masks are really on: the gradients differ from those without stochastic depth
    model = FSDPViT(tiny_cfg(mlp_dropout=0.1, att_dropout=0.1, pos_dropout=0.1), dtype=torch.float32, seed=3)
    model.forward_backward(IMAGES, TARGET)
    ref = full_grads_of(model)
    assert any(not torch.allclose(ref[k], grads[0][k]) for k in ref)


def test_mlp_dropout_composes_with_drop_path_like_autograd():
    """Block backward with both element dropout (mlp) and drop path against autograd through the same ops."""
    cfg = tiny_cfg(drop_path_rate=0.6, mlp_dropout=0.2)
    B = 4
    p = vit.init_block_params(cfg, torch.Generator().manual_seed(0))
    x = torch.randn(B * cfg.num_patches, cfg.embed_dim)
    dy = torch.randn_like(x)
    ctx = vit.DropoutCtx(9)
    y, s = vit.block_forward(torch_ops, cfg, p, x, B, save=True, drop=ctx, block_idx=2)
    G = {k: torch.zeros_like(v) for k, v in p.items()}
    dx, _ = vit.block_backward(torch_ops, cfg, p, G, s, dy, dy.sum(0), B)

    pa = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    xa = x.clone().requires_grad_(True)
    sa, sm = (t.repeat_interleave(cfg.num_patches)[:, None] for t in s["dpath"])
    pm, keys, N, H, hd = cfg.mlp_dropout, s["masks"], cfg.num_patches, cfg.num_heads, cfg.head_dim

    def drop(t, k):  # the element mask of torch_ops.dropout, as a differentiable product
        return t * torch_ops.dropout(torch.ones_like(t), pm, k)

    h = F.layer_norm(xa, (cfg.embed_dim,), pa["norm1.weight"], pa["norm1.bias"], 1e-5)
    qkv = F.linear(h, pa["attn.qkv.weight"], pa["attn.qkv.bias"]).view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    att = ((qkv[0] @ qkv[1].transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1)
    a = (att @ qkv[2]).transpose(1, 2).reshape(B * N, -1)
    x1 = xa + drop(F.linear(a, pa["attn.proj.weight"], pa["attn.proj.bias"]) * sa, keys["proj"])
    h = F.layer_norm(x1, (cfg.embed_dim,), pa["norm2.weight"], pa["norm2.bias"], 1e-5)
    gg = drop(F.gelu(F.linear(h, pa["mlp.fc1.weight"], pa["mlp.fc1.bias"])), keys["fc1"])
    ya = x1 + drop(F.linear(gg, pa["mlp.fc2.weight"], pa["mlp.fc2.bias"]) * sm, keys["fc2"])
    ya.backward(dy)
    assert (s["dpath"][0] == 0).any() or (s["dpath"][1] == 0).any()
    assert torch.allclose(y, ya, atol=1e-5)
    assert torch.allclose(dx, xa.grad, atol=1e-5)
    for k in p:
        assert (G[k] - pa[k].grad).abs().max() <= 1e-4 * pa[k].grad.abs().max() + 1e-7, k


def test_sample_dropped_in_both_branches_passes_through():
    cfg = tiny_cfg(drop_path_rate=0.9, num_blocks=2)
    B = 16
    p = vit.init_block_params(cfg, torch.Generator().manual_seed(0))
    x = torch.randn(B * cfg.num_patches, cfg.embed_dim)
    y, s = vit.block_forward(torch_ops, cfg, p, x, B, save=True, drop=vit.DropoutCtx(2), block_idx=1)
    both = ((s["dpath"][0] == 0) & (s["dpath"][1] == 0)).nonzero().flatten().tolist()
    kept = ((s["dpath"][0] > 0) | (s["dpath"][1] > 0)).nonzero().flatten().tolist()
    assert both and kept
    xs, ys = x.view(B, cfg.num_patches, -1), y.view(B, cfg.num_patches, -1)
    for b in both:
        assert torch.equal(ys[b], xs[b])
    for b in kept:
        assert not torch.equal(ys[b], xs[b])


def test_eval_logits_equal_rate_zero():
    a = FSDPViT(tiny_cfg(drop_path_rate=0.3), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    assert torch.equal(a.eval()(IMAGES), b.eval()(IMAGES))
    # training mode does drop
    assert not torch.equal(a.train()(IMAGES), b.train()(IMAGES))


# ------------------------------------------------------------------------------------------------
# FSDP / data-parallel equivalence: masks are drawn at the global sample index
# ------------------------------------------------------------------------------------------------
def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.fixture(scope="module")
def dp_baseline(tmp_path_factory):
    out = tmp_path_factory.mktemp("dp_base") / "r.json"
    return launch(1, {"model": {"drop_path_rate": 0.3}, "steps": 4}, str(out))


def test_trajectory_differs_from_rate_zero(dp_baseline, tmp_path):
    plain = launch(1, {"steps": 4}, str(tmp_path / "r.json"))
    assert any(abs(a - b) > 1e-4 for a, b in zip(plain["losses"], dp_baseline["losses"]))


@pytest.mark.parametrize("world,opts", [(2, {}), (4, {}), (8, {}), (2, {"no_fsdp": True}), (1, {"no_fsdp": True})])
def test_same_trajectory_at_every_world_size(world, opts, dp_baseline, tmp_path):
    res = launch(world, dict(opts, model={"drop_path_rate": 0.3}, steps=4), str(tmp_path / "r.json"))
    _close(res["losses"], dp_baseline["losses"])
    _close(res["norms"], dp_baseline["norms"], tol=1e-4)


# ------------------------------------------------------------------------------------------------
# CLI / config
# ------------------------------------------------------------------------------------------------
def test_cli_parsing():
    assert parse_args([]).drop_path_rate == 0.0
    args = parse_args(["--drop_path_rate", "0.2"])
    assert args.drop_path_rate == 0.2
    assert ViTConfig.from_args(args).drop_path_rate == 0.2
    assert ViTConfig.from_args(parse_args([])).drop_path_rate == 0.0


@pytest.mark.parametrize("bad", ["-0.1", "1", "1.5", "nan"])
def test_cli_rejects_invalid_rates(bad):
    with pytest.raises(SystemExit):
        parse_args(["--drop_path_rate", bad])
    with pytest.raises(ValueError):
        ViTConfig(drop_path_rate=float(bad))


def test_cuda_graph_refuses_drop_path():
    model = FSDPViT(tiny_cfg(drop_path_rate=0.1), dtype=torch.float32, seed=3)
    with pytest.raises(RuntimeError, match="drop_path_rate"):
        GraphedTrainStep(model, ShardedAdamW(model, lr=1e-3))


# ------------------------------------------------------------------------------------------------
# build: the GEMM with the row-scale epilogue stays call-free and spill-free
# ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")),
                    reason="needs nvcc")
def test_gemm_compiles_for_sm90a_without_calls_or_spills(tmp_path):
    from vit_10b_fsdp_example_b200 import build_ext

    nvcc = os.path.join(build_ext._cuda_home(), "bin", "nvcc")
    res = subprocess.run([nvcc, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, "gemm_sm90.cu"), "-o", str(tmp_path / "g.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    log = res.stdout + res.stderr
    assert "C7510" not in log
    entries = [ln for ln in log.splitlines() if "Compiling entry function" in ln and "gemm_bf16_sm90_kernel" in ln]
    assert len(entries) >= 20 and all("sm_90a" in ln for ln in entries)
    assert sum("ELb1EE" in ln for ln in entries) == 4  # the row-scale instantiations: K-major A / B, 2 tiles x 2 clusters
    spills = [ln for ln in log.splitlines() if "spill stores" in ln]
    assert len(spills) >= 20
    assert all("0 bytes spill stores, 0 bytes spill loads" in ln for ln in spills), spills
    if shutil.which("cuobjdump"):
        sass = subprocess.run(["cuobjdump", "-sass", str(tmp_path / "g.o")], capture_output=True, text=True).stdout
        assert "gemm_bf16_sm90_kernel" in sass and " CALL" not in sass
