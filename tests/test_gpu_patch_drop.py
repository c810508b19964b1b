"""Patch dropout on the GPU: the selection kernel bit-exact against the NumPy reference, the gathered im2col, pos_gather
and patch_drop_bwd against torch_ops and fp64, their argument checks, and the model with --patch_drop_rate against the
fp32 CPU model on both attention routes, across activation-keeping modes and through the command line."""
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
KEY = 0x1234_5678_9ABC_DEF


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _to():
    from vit_10b_fsdp_example_b200.ops import torch_ops

    return torch_ops


@pytest.mark.parametrize("N", [49, 196, 256, 1369, 4096])
@pytest.mark.parametrize("B,offset", [(1, 0), (6, 0), (7, 13), (4, 2 ** 31 + 5)])
def test_select_is_bit_exact_against_numpy(N, B, offset):
    co, to = _co(), _to()
    for K in sorted({1, N // 4, N // 2, N - 1, N} - {0}):
        keep, inv = co.patch_drop_select(KEY + N, B, N, K, offset, "cuda")
        rk, ri = to.patch_drop_select(KEY + N, B, N, K, offset, "cpu")
        torch.cuda.synchronize()
        assert torch.equal(keep.cpu(), rk), (N, K, B, offset)
        assert torch.equal(inv.cpu(), ri), (N, K, B, offset)


@pytest.mark.parametrize("mix", [None, (0.3, None), (0.6, (20, 150, 33, 201))])
@pytest.mark.parametrize("img_dtype", [torch.float32, torch.bfloat16])
def test_gathered_im2col_and_pos_gather_are_bitwise(mix, img_dtype):
    co, to = _co(), _to()
    B, S, P, kpad, D = 6, 224, 14, 592, 320
    g = torch.Generator().manual_seed(1)
    images = torch.randn(B, 3, S, S, generator=g).to(img_dtype)
    keep, _ = co.patch_drop_select(KEY, B, 256, 100, 3, "cuda")
    cols = co.patch_im2col(images.cuda(), P, kpad, torch.bfloat16, mix=mix, keep=keep)
    full = co.patch_im2col(images.cuda(), P, kpad, torch.bfloat16, mix=mix)
    ref = to.patch_im2col(images.float(), P, kpad, torch.bfloat16, mix=mix, keep=keep.cpu())
    rows = (torch.arange(B, device="cuda")[:, None] * 256 + keep.long()).reshape(-1)
    assert torch.equal(cols, full[rows])
    assert torch.equal(cols.cpu(), ref)
    pos = torch.randn(256, D, generator=g).bfloat16()
    out = co.pos_gather(pos.cuda(), keep)
    assert torch.equal(out.cpu(), to.pos_gather(pos, keep.cpu()))


@pytest.mark.parametrize("B,N,K,P,D", [(128, 256, 128, 0, 5120), (128, 256, 128, 1, 5120), (5, 49, 24, 5, 64),
                                       (3, 4096, 1, 2, 8), (8, 196, 196, 1, 136)])
def test_patch_drop_bwd_against_fp64_and_reproducible(B, N, K, P, D):
    co, to = _co(), _to()
    g = torch.Generator().manual_seed(N + P)
    keep, inv = co.patch_drop_select(KEY, B, N, K, 0, "cuda")
    dx0 = (torch.randn(B * (P + K), D, generator=g) * 4).bfloat16().cuda()
    dpatch, dtok = co.patch_drop_bwd(dx0, inv, B, N, K, P)
    dpatch2, dtok2 = co.patch_drop_bwd(dx0, inv, B, N, K, P)
    torch.cuda.synchronize()
    assert torch.equal(dtok, dtok2)  # b = 0 .. B-1 in order, no atomics
    x = dx0.view(B, P + K, D)
    if P:
        assert torch.equal(dpatch, x[:, P:].reshape(B * K, D)) and torch.equal(dpatch, dpatch2)
    else:
        assert dpatch is None
    xd = x.double().cpu()
    kp = keep.long().cpu()
    want = torch.zeros(P + N, D, dtype=torch.float64)
    mag = torch.zeros(P + N, D, dtype=torch.float64)
    want[:P], mag[:P] = xd[:, :P].sum(0), xd[:, :P].abs().sum(0)
    want[P:].index_add_(0, kp.reshape(-1), xd[:, P:].reshape(-1, D))
    mag[P:].index_add_(0, kp.reshape(-1), xd[:, P:].reshape(-1, D).abs())
    # at most B fp32 additions per entry, each rounding by <= 2^-24 of a partial sum bounded by sum |terms|
    assert ((dtok.double().cpu() - want).abs() <= B * 2.0 ** -24 * mag).all()


def test_rejects_bad_arguments():
    co = _co()
    C = co._C
    keep = torch.zeros(2, 4, dtype=torch.int32, device="cuda")
    inv = torch.zeros(2, 8, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="1 <= K <= N"):
        C.patch_drop_select(torch.zeros(2, 9, dtype=torch.int32, device="cuda"), inv, 8, 9, 0, 1)
    with pytest.raises(RuntimeError, match="N <= 4096"):
        C.patch_drop_select(torch.zeros(1, 4, dtype=torch.int32, device="cuda"),
                            torch.zeros(1, 4097, dtype=torch.int32, device="cuda"), 4097, 4, 0, 1)
    with pytest.raises(RuntimeError, match="int32"):
        C.patch_drop_select(keep.long(), inv, 8, 4, 0, 1)
    with pytest.raises(RuntimeError, match="2\\^32"):
        C.patch_drop_select(keep, inv, 8, 4, 2 ** 32 - 1, 1)
    pos = torch.zeros(8, 12, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="D % 8"):
        C.pos_gather(pos, keep, torch.zeros(8, 12, dtype=torch.bfloat16, device="cuda"))
    buf = torch.zeros(8 * 16 + 1, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        C.pos_gather(buf[1:].view(8, 16), keep, torch.zeros(8, 16, dtype=torch.bfloat16, device="cuda"))
    dtok = torch.zeros(1 + 8, 16, device="cuda")
    with pytest.raises(RuntimeError, match="dx0"):
        C.patch_drop_bwd(torch.zeros(2 * 4, 16, dtype=torch.bfloat16, device="cuda"), inv, None, dtok, 2, 8, 4, 1)
    with pytest.raises(RuntimeError, match="1 <= K <= N"):
        C.patch_drop_bwd(torch.zeros(2 * 10, 16, dtype=torch.bfloat16, device="cuda"), inv, None, dtok, 2, 8, 9, 1)
    img = torch.zeros(2, 3, 32, 32, device="cuda")
    with pytest.raises(RuntimeError, match="cols"):
        C.im2col_gather(img, keep, torch.zeros(7, 200, dtype=torch.bfloat16, device="cuda"), 8)
    with pytest.raises(RuntimeError, match="even batch"):
        C.im2col_gather(torch.zeros(1, 3, 32, 32, device="cuda"), keep[:1], torch.zeros(4, 200, dtype=torch.bfloat16,
                                                                                        device="cuda"), 8, 0.5)
    torch.cuda.synchronize()


def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=3, mlp_ratio=4.0, num_classes=96,
             patch_drop_rate=0.5)
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
    from helpers import full_params_of

    g = torch.Generator().manual_seed(seed)
    full = {k: v.cpu() for k, v in full_params_of(model).items()}
    for k in ("cls_token", "reg_token", "pos_embed"):
        if k in full:
            full[k] = torch.randn(full[k].shape, generator=g)
    model.load_full_state_dict(full)


@pytest.mark.parametrize("route,kw", [("fused", dict()), ("fused", dict(patch_drop_rate=0.25, qk_norm=True)),
                                      ("unfused", dict(class_token=True)),
                                      ("unfused", dict(class_token=True, reg_tokens=4, no_embed_class=True,
                                                       mixup=0.8, smoothing=0.1))])
def test_model_matches_the_fp32_cpu_model(route, kw):
    """bf16 GPU vs fp32 CPU loss and gradients with the same kept patches (the selection is bit-exact).  fused: no
    class token, T' = 128 or 192 (even: the wgmma attention pair); unfused: T' = 129 or 133 (odd)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg(**kw)
    assert cuda_ops.use_flash(cfg.train_tokens, cfg.head_dim) == (route == "fused"), cfg.train_tokens
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
        for k in g_ref:
            a, b = g_ref[k], grads[k]
            if k.endswith("k_norm.bias"):  # zero in exact arithmetic (the softmax cancels q . b_k): rounding is left
                ref = g_ref[k.replace("k_norm.bias", "qkv.bias")].norm().item()
                assert b.norm().item() <= 1e-3 * ref, (keep, k, b.norm().item(), ref)
                continue
            # bf16 activations and weights through three blocks: 5 % of the gradient's norm, as for the other flags
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (keep, k)


@pytest.mark.parametrize("kw", [dict(), dict(class_token=True, reg_tokens=2, pos_dropout=0.1, drop_path_rate=0.5)])
def test_checkpointed_kept_and_uncheckpointed_blocks_give_the_same_gradients(kw):
    """GEMM-produced weight gradients are bitwise equal; column sums reduced with fp32 atomics differ by at most one
    bf16 ulp (as in the other features' tests)."""
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
                assert torch.equal(g0[k], g1[k]), (k, diff)
            else:
                one_ulp = g0[k].abs() * 2.0 ** -7 + 1e-6 * g0[k].abs().max().item()
                assert ((g0[k] - g1[k]).abs() <= one_ulp).all(), (k, diff)


def test_cli_trains_checkpoints_consolidates_and_evaluates_with_patch_dropout(tmp_path):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "16",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--num_epochs", "1", "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--class_token",
            "--patch_drop_rate", "0.5"]
    ckpt = tmp_path / "ckpt"
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(ckpt)], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "patch_drop_rate=0.5" in r.stdout
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
    assert re.search(r"accuracy on val: [0-9.]+", r.stdout), r.stdout[-2000:]
    full = consolidate_files(str(ckpt / "epoch_1"))
    assert full["pos_embed"].shape == (1, 1 + 196, 128)
    cfg = ViTConfig(image_size=224, patch_size=16, embed_dim=128, num_heads=2, num_blocks=2, num_classes=10,
                    class_token=True, patch_drop_rate=0.5)
    plain = PlainViT(cfg)
    plain.load_state_dict(full, strict=True)
    with torch.no_grad():
        assert torch.isfinite(plain.eval()(torch.randn(2, 3, 224, 224))).all()
