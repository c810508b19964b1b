"""Mixup / CutMix fused into the patch im2col and the soft-target cross-entropy kernel, on the GPU.

torch_ops (a timm 0.4.12 transcription, fp32) is the reference: the im2col must match it bit for bit, the loss to fp32
rounding and dlogits to bf16 rounding."""
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
DEIT = dict(mixup=0.8, cutmix=1.0, smoothing=0.1)


def _ops():
    from vit_10b_fsdp_example_b200.ops import cuda_ops, torch_ops

    return cuda_ops, torch_ops


S = 224
MIXES = {
    "mixup_0.3": (0.3, None),
    "mixup_odd": (0.6180339887498949, None),
    "mixup_0": (0.0, None),
    "cutmix_inside": (0.5, (37, 150, 60, 141)),
    "cutmix_top": (0.5, (0, 90, 20, 200)),
    "cutmix_bottom": (0.5, (101, S, 3, 77)),
    "cutmix_left": (0.5, (50, 60, 0, 130)),
    "cutmix_right": (0.5, (1, 223, 112, S)),
    "cutmix_empty": (0.5, (80, 80, 10, 100)),
    "cutmix_whole": (0.0, (0, S, 0, S)),
}


@pytest.mark.parametrize("name", sorted(MIXES))
@pytest.mark.parametrize("img_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B,P", [(2, 16), (4, 32), (4, 14), (128, 14)])
def test_im2col_mix_is_bitwise_the_reference(name, img_dtype, B, P):
    co, to = _ops()
    mix = MIXES[name]
    g = torch.Generator().manual_seed(B * 100 + P)
    images = torch.randn(B, 3, S, S, generator=g).to(img_dtype)
    kpad = (3 * P * P + 7) // 8 * 8
    got = co.patch_im2col(images.cuda(), P, kpad, torch.bfloat16, mix=mix).cpu()
    want = to.patch_im2col(images, P, kpad, torch.bfloat16, mix=mix)
    assert torch.equal(got, want), (got.float() - want.float()).abs().max()
    plain = co.patch_im2col(images.cuda(), P, kpad, torch.bfloat16).cpu()
    assert torch.equal(plain, to.patch_im2col(images, P, kpad, torch.bfloat16))
    if name in ("cutmix_empty",):
        assert torch.equal(got, plain)


def test_im2col_rejects_bad_mixes():
    co, _ = _ops()
    x = torch.randn(3, 3, 32, 32, device="cuda")
    with pytest.raises(RuntimeError, match="even batch"):
        co.patch_im2col(x, 8, 192, torch.bfloat16, mix=(0.5, None))
    with pytest.raises(RuntimeError, match="inside the image"):
        co.patch_im2col(x[:2], 8, 192, torch.bfloat16, mix=(0.5, (0, 33, 0, 4)))


@pytest.mark.parametrize("mix,s", [((0.3, None), 0.0), ((0.77, (1, 2, 3, 4)), 0.0), (None, 0.1), ((0.3, None), 0.1),
                                   ((0.0, None), 0.2)])
@pytest.mark.parametrize("B", [2, 128])
@pytest.mark.parametrize("C", [10, 1000, 1001])
def test_soft_cross_entropy_matches_the_fp32_reference(mix, s, B, C):
    co, to = _ops()
    g = torch.Generator().manual_seed(B + C)
    logits = (torch.randn(B, C, generator=g) * 3).to(torch.bfloat16)
    target = torch.randint(0, C, (B,), generator=g)
    target[0] = target[-1]
    loss, dl, correct = co.cross_entropy(logits.cuda(), target.cuda(), want_grad=True, mix=mix, smoothing=s)
    rl, rdl, rc = to.cross_entropy(logits.float(), target, want_grad=True, mix=mix, smoothing=s)
    assert abs(loss.item() - rl.item()) <= 1e-4 * abs(rl.item()) + 1e-5, (loss.item(), rl.item())
    err = (dl.float().cpu() - rdl).abs()
    assert (err <= rdl.abs() * 2 ** -7 + 1e-5 / B).all(), err.max().item()
    assert correct.item() == rc.item()


@pytest.mark.parametrize("C", [10, 1000, 1001])
def test_lam_one_smoothing_zero_is_bitwise_the_hard_call(C):
    co, _ = _ops()
    g = torch.Generator().manual_seed(C)
    B = 16
    logits = (torch.randn(B, C, generator=g) * 3).to(torch.bfloat16).cuda()
    target = torch.randint(0, C, (B,), generator=g).cuda()

    def run(*extra):
        loss = torch.zeros(1, device="cuda")
        correct = torch.zeros(1, dtype=torch.int32, device="cuda")
        dl = torch.empty_like(logits)
        co._C.cross_entropy(logits, target, dl, loss, correct, *extra)
        return loss, dl, correct

    hard, soft = run(), run(1.0, 0.0)
    assert torch.equal(hard[1], soft[1]) and torch.equal(hard[2], soft[2])
    for r in range(B):  # one row per call: a single atomic add, so the loss bits are reproducible
        lh = torch.zeros(1, device="cuda")
        ls = torch.zeros(1, device="cuda")
        co._C.cross_entropy(logits[r:r + 1], target[r:r + 1], None, lh, None)
        co._C.cross_entropy(logits[r:r + 1], target[r:r + 1], None, ls, None, 1.0, 0.0)
        assert torch.equal(lh, ls), r


# ------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=2, mlp_ratio=4.0, num_classes=96,
             **DEIT)
    d.update(kw)
    return ViTConfig(**d)


def _full_grads(model):
    out = {}
    for u in model.all_units:
        for n, v in u.layout.param_views(u.shard_grad.float()).items():
            out[f"{u.name}.{n}"] = v.detach().cpu().clone()
    return out


def test_model_step_matches_the_fp32_cpu_model():
    """bf16 GPU model vs fp32 CPU model at the same step counts, so both draw the same Mixup / CutMix parameters."""
    from vit_10b_fsdp_example_b200.models import vit
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg()
    draws = {s: vit.draw_mix(cfg, vit.mix_rng(4, s, 0)) for s in range(40)}
    steps = [next(s for s, d in draws.items() if d is not None and d[1] is None),
             next(s for s, d in draws.items() if d is not None and d[1] is not None)]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(8, 3, 224, 224, generator=g)
    y = torch.randint(0, 96, (8,), generator=g)
    for step in steps:
        res = []
        for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
            model = FSDPViT(cfg, device=dev, dtype=dtype, seed=4)
            model.step_count = step
            loss = model.forward_backward(x.to(dev), y.to(dev)).item()
            res.append((loss, _full_grads(model)))
        (loss_ref, g_ref), (loss, grads) = res
        assert math.isfinite(loss) and abs(loss - loss_ref) < 1e-2 * abs(loss_ref) + 1e-2, (step, loss, loss_ref)
        for k in g_ref:
            a, b = g_ref[k], grads[k]
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (step, k)


def test_cuda_graph_with_smoothing_matches_eager():
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

    cfg = _cfg(image_size=112, embed_dim=320, num_heads=2, mixup=0.0, cutmix=0.0, smoothing=0.1)
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
            assert step.graph is not None
    for a, b in zip(results["eager"], results["graph"]):
        assert abs(a - b) < 2e-2 * abs(a) + 1e-3, results


def test_cli_trains_with_mixup_cutmix_smoothing_on_an_image_folder(tmp_path):
    from PIL import Image

    g = torch.Generator().manual_seed(0)
    for split, per_class in (("train", 16), ("val", 4)):
        for c, cls in enumerate(("n01", "n02")):
            d = tmp_path / "data" / split / cls
            d.mkdir(parents=True)
            for i in range(per_class):
                arr = (torch.rand(40, 48, 3, generator=g) * 80 + 160 * c).to(torch.uint8).numpy()
                Image.fromarray(arr).save(d / f"img_{i}.jpeg")
    args = ["--data_dir", str(tmp_path / "data"), "--device", "cuda", "--nproc", "1", "--image_size", "224",
            "--patch_size", "16", "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "2",
            "--batch_size", "8", "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1",
            "--num_workers", "0", "--num_epochs", "1", "--ckpt_epoch_interval", "100", "--test_epoch_interval", "100",
            "--mixup", "0.8", "--cutmix", "1.0", "--smoothing", "0.1"]
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(tmp_path / "ckpt")], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
