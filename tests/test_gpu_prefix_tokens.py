"""Class and register tokens on the GPU: the tokens_fwd / tokens_bwd kernels against fp64 references computed from the
same bf16 inputs, their argument checks, and the model with --class_token against the fp32 CPU model on both attention
routes, across activation-keeping modes, under CUDA graphs and through the command line.

Tolerances are derived from the kernels' arithmetic and written beside each check."""
import math
import os
import re
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32_EPS = 2.0 ** -24  # unit roundoff of fp32


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _inputs(B, N, P, D, embed, seed):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(B * N, D, generator=g).bfloat16().cuda()
    cls = torch.randn(1, D, generator=g).bfloat16().cuda()
    reg = torch.randn(P - 1, D, generator=g).bfloat16().cuda() if P > 1 else None
    pos = torch.randn(P, D, generator=g).bfloat16().cuda() if embed else None
    dx0 = (torch.randn(B * (N + P), D, generator=g) * torch.rand(B * (N + P), 1, generator=g) * 4).bfloat16().cuda()
    return y, cls, reg, pos, dx0


def _check(B, N, P, D, embed, seed=0):
    co = _co()
    y, cls, reg, pos, dx0 = _inputs(B, N, P, D, embed, seed)
    T = N + P
    x0 = co.tokens_fwd(y, cls, reg, pos, B, N)
    dpatch, dtok = co.tokens_bwd(dx0, B, N, P)
    torch.cuda.synchronize()
    x = x0.view(B, T, D)
    # patch rows: a copy, bitwise
    assert torch.equal(x[:, P:], y.view(B, N, D))
    # prefix rows: the same IEEE fp32 add of two bf16 values and one rounding to bf16 as on the host -> bitwise equal;
    # and within half a bf16 ulp (bf16 keeps 8 significant bits: <= 2^-8 relative) plus the fp32 add's 2^-24 of the
    # exact fp64 sum
    pre = torch.cat([cls.float()] + ([reg.float()] if reg is not None else []))
    if pos is not None:
        pre = pre + pos.float()
    want = pre.bfloat16()
    for b in range(B):
        assert torch.equal(x[b, :P], want), b
    exact = torch.cat([cls.double()] + ([reg.double()] if reg is not None else [])) + (
        pos.double() if pos is not None else 0)
    assert ((x[0, :P].double() - exact).abs() <= (2.0 ** -8 + 2.0 ** -24) * exact.abs() + 1e-30).all()
    # dpatch: a copy, bitwise
    assert torch.equal(dpatch, dx0.view(B, T, D)[:, P:].reshape(B * N, D))
    # dtok: B - 1 fp32 additions in sequence: |err| <= (B - 1) eps32 * sum_b |dx0| (first-order bound)
    d = dx0.double().view(B, T, D)
    ref = d.sum(0)
    tol = (B - 1) * F32_EPS * d.abs().sum(0) + 1e-30
    err = (dtok.double() - ref).abs()
    worst = err.flatten().argmax()
    assert (err <= tol).all(), f"dtok: worst err {err.max().item():.3g}, tol there {tol.flatten()[worst].item():.3g}"
    return dx0, dtok


@pytest.mark.parametrize("P", [1, 5])
@pytest.mark.parametrize("embed", [True, False])
def test_kernels_at_the_vit10b_shape(P, embed):
    _check(128, 256, P, 5120, embed, seed=P)


@pytest.mark.parametrize("B,N,P,D", [(3, 9, 1, 72), (3, 9, 2, 72), (1, 1, 1, 8), (5, 7, 5, 24), (2, 225, 1, 320),
                                     (7, 49, 4, 16392), (33, 3, 3, 8)])
@pytest.mark.parametrize("embed", [True, False])
def test_kernels_at_small_and_odd_shapes(B, N, P, D, embed):
    _check(B, N, P, D, embed, seed=B * 1000 + N * 10 + P)


def test_tokens_bwd_is_bitwise_reproducible():
    co = _co()
    _, _, _, _, dx0 = _inputs(128, 256, 5, 5120, True, seed=3)
    a = co.tokens_bwd(dx0, 128, 256, 5)
    b = co.tokens_bwd(dx0, 128, 256, 5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_rejects_bad_arguments():
    co = _co()
    from vit_10b_fsdp_example_b200.ops import native

    C = native.load()
    B, N, P, D = 2, 4, 3, 16
    y, cls, reg, pos, dx0 = _inputs(B, N, P, D, True, seed=0)
    x0 = torch.empty(B * (N + P), D, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="tokens_fwd: y must be a bf16 CUDA tensor"):
        co.tokens_fwd(y.float(), cls, reg, pos, B, N)
    with pytest.raises(RuntimeError, match="tokens_fwd: cls must be a bf16 CUDA tensor"):
        co.tokens_fwd(y, cls.float(), reg, pos, B, N)
    with pytest.raises(RuntimeError, match=r"tokens_fwd: need D % 8 == 0"):
        co.tokens_fwd(y[:, :12].contiguous(), cls[:, :12].contiguous(), None, None, B, N)
    with pytest.raises(RuntimeError, match="tokens_fwd: y must be contiguous with 96 elements"):
        co.tokens_fwd(y, cls, reg, pos, B, N - 1)
    with pytest.raises(RuntimeError, match="tokens_fwd: pos must be contiguous with 48 elements"):
        co.tokens_fwd(y, cls, reg, pos[:2], B, N)
    with pytest.raises(RuntimeError, match="tokens_fwd: x0 must be contiguous with"):
        C.tokens_fwd(y, cls, reg, pos, x0[:-1], B, N)
    with pytest.raises(RuntimeError, match="tokens_fwd: x0 must be a bf16 CUDA tensor"):
        C.tokens_fwd(y, cls, reg, pos, x0.float(), B, N)
    buf = torch.empty(B * N * D + 4, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="tokens_fwd: y must be 16-byte aligned"):
        co.tokens_fwd(buf[4:].view(B * N, D), cls, reg, pos, B, N)
    with pytest.raises(RuntimeError, match="tokens_bwd: need P >= 1 prefix tokens"):
        co.tokens_bwd(dx0[: B * N], B, N, 0)
    with pytest.raises(RuntimeError, match="tokens_bwd: dx0 must be a bf16 CUDA tensor"):
        co.tokens_bwd(dx0.float(), B, N, P)
    with pytest.raises(RuntimeError, match="tokens_bwd: dx0 must be contiguous with"):
        co.tokens_bwd(dx0, B, N, P + 1)
    with pytest.raises(RuntimeError, match=r"tokens_bwd: need D % 8 == 0"):
        co.tokens_bwd(dx0[:, :12].contiguous(), B, N, P)
    dpatch = torch.empty(B * N, D, dtype=torch.bfloat16, device="cuda")
    dtok = torch.empty(N + P, D, dtype=torch.float32, device="cuda")
    with pytest.raises(RuntimeError, match="tokens_bwd: dtok must be a contiguous fp32 CUDA tensor"):
        C.tokens_bwd(dx0, dpatch, dtok[:-1], B, N, P)
    with pytest.raises(RuntimeError, match="tokens_bwd: dtok must be a contiguous fp32 CUDA tensor"):
        C.tokens_bwd(dx0, dpatch, dtok.bfloat16(), B, N, P)
    with pytest.raises(RuntimeError, match="tokens_bwd: dpatch must be contiguous with"):
        C.tokens_bwd(dx0, dpatch[:-1], dtok, B, N, P)
    buf = torch.empty(B * (N + P) * D + 4, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="tokens_bwd: dx0 must be 16-byte aligned"):
        co.tokens_bwd(buf[4:].view(B * (N + P), D), B, N, P)


# ------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=3, mlp_ratio=4.0, num_classes=96,
             class_token=True)
    d.update(kw)
    return ViTConfig(**d)


def _data(cfg, B=8):
    g = torch.Generator().manual_seed(0)
    return (torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=g),
            torch.randint(0, cfg.num_classes, (B,), generator=g))


def _named_grads(model):
    out = {}
    for u in model.all_units:  # world 1: the shard buffer has the full layout
        for n, v in u.layout.param_views(u.shard_grad.float()).items():
            out[f"{u.name}.{n}"] = v.detach().cpu().clone()
    return out


def _randomize(model, seed=0):
    """Prefix tokens and pos_embed at magnitude 1: at their 1e-6 start a wrong gradient would barely show."""
    from helpers import full_params_of

    g = torch.Generator().manual_seed(seed)
    full = {k: v.cpu() for k, v in full_params_of(model).items()}
    for k in ("cls_token", "reg_token", "pos_embed"):
        if k in full:
            full[k] = torch.randn(full[k].shape, generator=g)
    model.load_full_state_dict(full)


@pytest.mark.parametrize("route,kw", [("unfused", dict()), ("unfused", dict(reg_tokens=4, no_embed_class=True)),
                                      ("fused", dict(image_size=210)), ("fused", dict(image_size=210, reg_tokens=2))])
def test_model_matches_the_fp32_cpu_model(route, kw):
    """Same parameters (host init, random prefix tokens): bf16 GPU vs fp32 CPU loss and gradients.  unfused: T = 257
    or 261 (odd: the GEMM + softmax route, as at the ViT-10B grid with a class token); fused: T = 226 or 228 (15 x 15
    patches plus the prefix tokens: even T takes the wgmma attention pair)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg(**kw)
    assert cuda_ops.use_flash(cfg.num_tokens, cfg.head_dim) == (route == "fused"), cfg.num_tokens
    x, y = _data(cfg)
    for keep in (0, 3):
        res = []
        for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
            model = FSDPViT(cfg, device=dev, dtype=dtype, seed=4, ckpt_keep_blocks=keep)
            _randomize(model)
            loss = model.forward_backward(x.to(dev), y.to(dev)).item()
            res.append((loss, _named_grads(model)))
        (loss_ref, g_ref), (loss, grads) = res
        assert math.isfinite(loss) and abs(loss - loss_ref) < 1e-2 * abs(loss_ref) + 1e-2, (keep, loss, loss_ref)
        assert "root.cls_token" in g_ref
        for k in g_ref:
            a, b = g_ref[k], grads[k]
            # bf16 activations and weights through three blocks: 5 % of the gradient's norm, as for the other flags
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (keep, k)


@pytest.mark.parametrize("kw", [dict(), dict(image_size=210, reg_tokens=1), dict(att_dropout=0.1, mlp_dropout=0.1,
                                                                                    pos_dropout=0.1),
                                dict(drop_path_rate=0.5, qk_norm=True, init_values=1e-5, reg_tokens=4)])
def test_checkpointed_kept_and_uncheckpointed_blocks_give_the_same_gradients(kw):
    """GEMM-produced weight gradients are bitwise equal.  Biases and LayerNorm parameters come from column sums reduced
    with fp32 atomics in arrival order, whose last bits vary from run to run: one bf16 ulp.  The prefix-token, pos_embed
    and patch-bias gradients (tokens_bwd, fixed order) are held to the same bound."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg(**kw)
    x, y = _data(cfg)
    runs = []
    for mkw in (dict(grad_ckpt=True, ckpt_keep_blocks=0), dict(grad_ckpt=True, ckpt_keep_blocks=3),
                dict(grad_ckpt=False)):
        model = FSDPViT(cfg, device="cuda", dtype=torch.bfloat16, seed=4, **mkw)
        if mkw.get("ckpt_keep_blocks") == 3:
            model.keep_extras = {"P": 1, "h": 2, "g": 3}
        _randomize(model)
        runs.append((model.forward_backward(x.cuda(), y.cuda()).item(), _named_grads(model)))
    (l0, g0) = runs[0]
    for l1, g1 in runs[1:]:
        assert abs(l0 - l1) <= 1e-6 * abs(l0), (l0, l1)
        for k in g0:
            diff = (g0[k] - g1[k]).abs().max().item()
            if k.endswith(("qkv.weight", "proj.weight", "fc1.weight", "fc2.weight", "head.weight")):
                assert torch.equal(g0[k], g1[k]), (k, diff, g0[k].abs().max().item())
            elif k.endswith("k_norm.bias"):  # zero in exact arithmetic: rounding on the scale of the largest entry
                assert diff <= 2.0 ** -7 * g0[k].abs().max().item() + 1e-12, (k, diff)
            else:
                one_ulp = g0[k].abs() * 2.0 ** -7 + 1e-6 * g0[k].abs().max().item()  # bf16: 8 significant bits
                assert ((g0[k] - g1[k]).abs() <= one_ulp).all(), (k, diff, g0[k].abs().max().item())


def test_cuda_graph_matches_eager():
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

    cfg = _cfg(image_size=112, embed_dim=320, num_heads=2, reg_tokens=4)
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    images = [torch.randn(8, 3, 112, 112, generator=g).to(dev) for _ in range(3)]
    targets = [torch.randint(0, 96, (8,), generator=g).to(dev) for _ in range(3)]
    results = {}
    for mode in ("eager", "graph"):
        model = FSDPViT(cfg, device=dev, dtype=torch.bfloat16, seed=4)
        opt = ShardedAdamW(model, lr=1e-3, weight_decay=0.1)
        step = GraphedTrainStep(model, opt, clip_grad_norm=1.0, warmup=2) if mode == "graph" else None
        losses = []
        for i in range(6):
            x, y = images[i % 3], targets[i % 3]
            if step is not None:
                loss = step(x, y)
            else:
                loss = model.forward_backward(x, y)
                model.clip_grad_norm_(1.0)
                opt.step()
            losses.append(loss.item())
        results[mode] = losses
        if step is not None:
            assert step.graph is not None and step.launches_per_step > 0
    for a, b in zip(results["eager"], results["graph"]):
        assert abs(a - b) < 2e-2 * abs(a) + 1e-3, results


def test_cli_trains_checkpoints_consolidates_and_evaluates_with_class_token(tmp_path):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "16",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--num_epochs", "1", "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--class_token",
            "--reg_tokens", "2"]
    ckpt = tmp_path / "ckpt"
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(ckpt)], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "class_token=True" in r.stdout and "reg_tokens=2" in r.stdout
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
    assert re.search(r"accuracy on val: [0-9.]+", r.stdout), r.stdout[-2000:]
    full = consolidate_files(str(ckpt / "epoch_1"))
    assert full["cls_token"].shape == (1, 1, 128) and full["reg_token"].shape == (1, 2, 128)
    assert full["pos_embed"].shape == (1, 3 + 196, 128)
    cfg = ViTConfig(image_size=224, patch_size=16, embed_dim=128, num_heads=2, num_blocks=2, num_classes=10,
                    class_token=True, reg_tokens=2)
    plain = PlainViT(cfg)
    plain.load_state_dict(full, strict=True)
    with torch.no_grad():
        assert torch.isfinite(plain.eval()(torch.randn(2, 3, 224, 224))).all()
