"""Mixup, CutMix and label smoothing (--mixup / --cutmix / --smoothing): timm 0.4.12 draws, mixing and soft-target loss.

The references are line-by-line transcriptions of timm 0.4.12 (timm/data/mixup.py and timm/loss/cross_entropy.py),
driven by the same NumPy generator as the model's draw function.  The GPU kernels are held to torch_ops in
test_gpu_mixup.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dist_worker import launch
from helpers import full_grads_of, full_params_of, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.models.plain import PlainViT
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEIT = dict(mixup=0.8, cutmix=1.0, smoothing=0.1)


# ------------------------------------------------------------------------------------------------
# timm 0.4.12 transcription (np.random.rand / beta / randint -> the generator's random / beta / integers)
# ------------------------------------------------------------------------------------------------
def timm_params_per_batch(rng, mixup_alpha, cutmix_alpha, mix_prob, switch_prob):
    lam = 1.
    use_cutmix = False
    if rng.random() < mix_prob:
        if mixup_alpha > 0. and cutmix_alpha > 0.:
            use_cutmix = rng.random() < switch_prob
            lam_mix = rng.beta(cutmix_alpha, cutmix_alpha) if use_cutmix else \
                rng.beta(mixup_alpha, mixup_alpha)
        elif mixup_alpha > 0.:
            lam_mix = rng.beta(mixup_alpha, mixup_alpha)
        elif cutmix_alpha > 0.:
            use_cutmix = True
            lam_mix = rng.beta(cutmix_alpha, cutmix_alpha)
        else:
            assert False, "One of mixup_alpha > 0., cutmix_alpha > 0., cutmix_minmax not None should be true."
        lam = float(lam_mix)
    return lam, use_cutmix


def timm_rand_bbox(rng, img_shape, lam, margin=0.):
    ratio = np.sqrt(1 - lam)
    img_h, img_w = img_shape[-2:]
    cut_h, cut_w = int(img_h * ratio), int(img_w * ratio)
    margin_y, margin_x = int(margin * cut_h), int(margin * cut_w)
    cy = rng.integers(0 + margin_y, img_h - margin_y)
    cx = rng.integers(0 + margin_x, img_w - margin_x)
    yl = np.clip(cy - cut_h // 2, 0, img_h)
    yh = np.clip(cy + cut_h // 2, 0, img_h)
    xl = np.clip(cx - cut_w // 2, 0, img_w)
    xh = np.clip(cx + cut_w // 2, 0, img_w)
    return yl, yh, xl, xh


def timm_cutmix_bbox_and_lam(rng, img_shape, lam, correct_lam=True):
    yl, yu, xl, xu = timm_rand_bbox(rng, img_shape, lam)
    if correct_lam:
        bbox_area = (yu - yl) * (xu - xl)
        lam = 1. - bbox_area / float(img_shape[-2] * img_shape[-1])
    return (yl, yu, xl, xu), lam


def timm_mix_batch(x, lam, use_cutmix, rng):
    """Mixup._mix_batch: returns (mixed x, lam) and, for the comparison, the box or None."""
    x = x.clone()
    if lam == 1.:
        return x, 1., None
    if use_cutmix:
        (yl, yh, xl, xh), lam = timm_cutmix_bbox_and_lam(rng, x.shape, lam)
        x[:, :, yl:yh, xl:xh] = x.flip(0)[:, :, yl:yh, xl:xh]
        return x, lam, (int(yl), int(yh), int(xl), int(xh))
    x_flipped = x.flip(0).mul_(1. - lam)
    x.mul_(lam).add_(x_flipped)
    return x, lam, None


def timm_one_hot(x, num_classes, on_value=1., off_value=0., device="cpu"):
    x = x.long().view(-1, 1)
    return torch.full((x.size()[0], num_classes), off_value, device=device).scatter_(1, x, on_value)


def timm_mixup_target(target, num_classes, lam=1., smoothing=0.0, device="cpu"):
    off_value = smoothing / num_classes
    on_value = 1. - smoothing + off_value
    y1 = timm_one_hot(target, num_classes, on_value=on_value, off_value=off_value, device=device)
    y2 = timm_one_hot(target.flip(0), num_classes, on_value=on_value, off_value=off_value, device=device)
    return y1 * lam + y2 * (1. - lam)


def timm_step(cfg, rng, images):
    """The whole timm Mixup.__call__ (mode 'batch') on a batch: mixed images, lam and box."""
    lam, use_cutmix = timm_params_per_batch(rng, cfg.mixup, cfg.cutmix, cfg.mixup_prob, cfg.mixup_switch_prob)
    return timm_mix_batch(images, lam, use_cutmix, rng)


# ------------------------------------------------------------------------------------------------
# draws
# ------------------------------------------------------------------------------------------------
CASES = {
    "mixup_only": dict(mixup=0.8),
    "cutmix_only": dict(cutmix=1.0),
    "both": dict(mixup=0.8, cutmix=1.0),
    "prob_below_1": dict(mixup=0.8, cutmix=1.0, mixup_prob=0.4, mixup_switch_prob=0.3),
    "small_alpha_cutmix": dict(cutmix=0.1),  # lam near 0 or 1: boxes clipped at the border or of zero area
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_draw_matches_timm_transcription(case):
    cfg = tiny_cfg(**CASES[case])
    img = torch.zeros(2, 3, cfg.image_size, cfg.image_size)
    seen = {"none": 0, "mixup": 0, "cutmix": 0, "clipped": 0, "corrected_to_1": 0}
    for step in range(300):
        for rank in (0, 3):
            got = vit.draw_mix(cfg, vit.mix_rng(5, step, rank))
            rng = vit.mix_rng(5, step, rank)
            lam_t, use_cutmix = timm_params_per_batch(rng, cfg.mixup, cfg.cutmix, cfg.mixup_prob,
                                                      cfg.mixup_switch_prob)
            _, lam, box = timm_mix_batch(img, lam_t, use_cutmix, rng)
            if lam == 1.:
                assert got is None, (step, rank, got)
                seen["none"] += 1
                seen["corrected_to_1"] += lam_t != 1. and use_cutmix
                continue
            assert got == (lam, box), (step, rank, got, lam, box)
            assert isinstance(got[0], float)
            seen["cutmix" if box else "mixup"] += 1
            if box:
                S = cfg.image_size
                seen["clipped"] += box[0] == 0 or box[1] == S or box[2] == 0 or box[3] == S
    if cfg.mixup > 0:
        assert seen["mixup"] > 0
    if cfg.cutmix > 0:
        assert seen["cutmix"] > 0 and seen["clipped"] > 0
    if cfg.mixup_prob < 1:
        assert seen["none"] > 100
    if case == "small_alpha_cutmix":
        assert seen["corrected_to_1"] > 0
    if case == "mixup_only":
        assert seen["none"] == 0


def test_no_draw_when_off_and_draws_differ_by_step_and_rank():
    assert vit.draw_mix(tiny_cfg(smoothing=0.1), vit.mix_rng(0, 0, 0)) is None
    cfg = tiny_cfg(mixup=0.8)
    draws = {(s, r): vit.draw_mix(cfg, vit.mix_rng(1, s, r)) for s in range(4) for r in range(2)}
    assert len({d[0] for d in draws.values()}) == len(draws)
    assert draws[(2, 1)] == vit.draw_mix(cfg, vit.mix_rng(1, 2, 1))


# ------------------------------------------------------------------------------------------------
# images and targets
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mix", [(0.3, None), (0.7071, None), (0.0, None), (0.6, (3, 20, 0, 32)), (0.9, (0, 0, 5, 9)),
                                 (0.0, (0, 32, 0, 32)), (0.75, (16, 32, 24, 32))])
def test_torch_ops_mixing_is_timm_mix_batch(mix):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(6, 3, 32, 32, generator=g)
    lam, box = mix
    if box is None:
        want = x.clone()
        want_f = want.flip(0).mul_(1. - lam)
        want.mul_(lam).add_(want_f)
    else:
        want = x.clone()
        want[:, :, box[0]:box[1], box[2]:box[3]] = x.flip(0)[:, :, box[0]:box[1], box[2]:box[3]]
    got = torch_ops.mix_images(x, mix)
    assert torch.equal(got, want)
    assert torch.equal(x, torch.randn(6, 3, 32, 32, generator=torch.Generator().manual_seed(3)))  # input untouched
    cols = torch_ops.patch_im2col(x, 8, 200, torch.float32, mix=mix)
    assert torch.equal(cols, torch_ops.patch_im2col(want, 8, 200, torch.float32))


LOSS_CASES = [(None, 0.0), (None, 0.1), ((0.3, None), 0.0), ((0.62, (1, 2, 3, 4)), 0.1), ((0.0, None), 0.2),
              ((1.0 - 2 ** -20, None), 0.0)]


@pytest.mark.parametrize("mix,s", LOSS_CASES)
@pytest.mark.parametrize("C", [10, 1000, 1001])
def test_loss_and_grad_equal_soft_target_cross_entropy(mix, s, C):
    g = torch.Generator().manual_seed(C)
    B = 8
    logits = torch.randn(B, C, generator=g, dtype=torch.float64).float() * 3
    target = torch.randint(0, C, (B,), generator=g)
    target[0] = target[-1]  # a pair with the same label
    lam = 1.0 if mix is None else mix[0]
    soft = timm_mixup_target(target, C, lam, s)
    lg = logits.clone().requires_grad_(True)
    ref = F.cross_entropy(lg, soft)  # probability targets: timm SoftTargetCrossEntropy
    ref.backward()
    loss, dlogits, correct = torch_ops.cross_entropy(logits, target, want_grad=True, mix=mix, smoothing=s)
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item()) + 1e-6
    assert torch.allclose(dlogits, lg.grad, atol=1e-7, rtol=1e-5)
    assert correct.item() == int((logits.argmax(-1) == target).sum())  # counted against y_b
    # the closed form the kernel computes
    off, on = s / C, 1 - s + s / C
    closed = (torch.logsumexp(logits.double(), -1) - off * logits.double().sum(-1)
              - (on - off) * (lam * logits.double().gather(1, target[:, None])[:, 0]
                              + (1 - lam) * logits.double().gather(1, target.flip(0)[:, None])[:, 0])).mean()
    assert abs(closed.item() - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-6
    if mix is None:  # label smoothing alone: DeiT LabelSmoothingCrossEntropy == F.cross_entropy(label_smoothing=s)
        assert abs(F.cross_entropy(logits, target, label_smoothing=s).item() - loss.item()) <= 1e-5


def test_hard_loss_path_is_unchanged():
    g = torch.Generator().manual_seed(1)
    logits, target = torch.randn(6, 10, generator=g), torch.randint(0, 10, (6,), generator=g)
    loss, d, c = torch_ops.cross_entropy(logits, target)
    assert torch.equal(loss, F.cross_entropy(logits, target)) or abs(loss - F.cross_entropy(logits, target)) < 1e-6
    loss1, d1, _ = torch_ops.cross_entropy(logits, target, mix=(1.0, None))
    assert abs(loss1.item() - loss.item()) < 1e-6 and torch.allclose(d1, d, atol=1e-8)


# ------------------------------------------------------------------------------------------------
# model step
# ------------------------------------------------------------------------------------------------
def _plain_from(model):
    cfg = model.cfg
    full = full_params_of(model)
    P, D = cfg.patch_size, cfg.embed_dim
    full["patch_embed.proj.weight"] = full["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(D, 3, P, P)
    full["pos_embed"] = full["pos_embed"].view(1, cfg.num_patches, D)
    return PlainViT.from_consolidated(full, cfg)


@pytest.mark.parametrize("kw,step", [(DEIT, 0), (DEIT, 1), (DEIT, 2), (dict(mixup=0.5), 0), (dict(cutmix=1.0), 3),
                                     (dict(smoothing=0.2), 0)])
def test_engine_step_equals_plain_vit_autograd_on_mixed_batch(kw, step):
    cfg = tiny_cfg(**kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3)
    model.step_count = step
    g = torch.Generator().manual_seed(11)
    images = torch.randn(6, 3, cfg.image_size, cfg.image_size, generator=g)
    target = torch.randint(0, cfg.num_classes, (6,), generator=g)
    target[1] = target[4]
    plain = _plain_from(model)
    # timm Mixup applied to the batch on the host, then SoftTargetCrossEntropy through autograd
    if cfg.mixing:
        xm, lam, _ = timm_step(cfg, vit.mix_rng(3, step, 0), images)
    else:
        xm, lam = images, 1.0
    soft = timm_mixup_target(target, cfg.num_classes, lam, cfg.smoothing)
    ref = torch.sum(-soft * F.log_softmax(plain(xm), dim=-1), dim=-1).mean()
    ref.backward()

    loss = model.forward_backward(images, target)
    assert model.step_count == step + 1
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    got = full_grads_of(model)
    want = {n: p.grad for n, p in plain.named_parameters()}
    for n, w in want.items():
        gn = got[n]
        if n == "patch_embed.proj.weight":
            gn = gn[:, : cfg.patch_k].reshape(w.shape)
        gn = gn.view(w.shape)
        assert (gn - w).abs().max().item() <= 2e-4 * w.abs().max().item() + 1e-7, n


def test_flags_zero_call_no_new_op(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("mixing drawn at flags 0")

    monkeypatch.setattr(vit, "draw_mix", boom)
    monkeypatch.setattr(vit, "mix_rng", boom)
    calls = []
    real_im2col, real_ce = torch_ops.patch_im2col, torch_ops.cross_entropy

    def im2col(*a, **k):
        calls.append(("im2col", len(a), tuple(k)))
        return real_im2col(*a, **k)

    def ce(*a, **k):
        calls.append(("ce", len(a), tuple(k)))
        return real_ce(*a, **k)

    monkeypatch.setattr(torch_ops, "patch_im2col", im2col)
    monkeypatch.setattr(torch_ops, "cross_entropy", ce)
    images, target = torch.randn(4, 3, 32, 32), torch.tensor([1, 5, 7, 2])
    for kw in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(run_without_fsdp=True)):
        FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3, **kw).forward_backward(images, target)
    assert calls and all(c in (("im2col", 4, ()), ("ce", 2, ("want_grad",))) for c in calls), calls


def test_no_mix_step_with_mixing_on_passes_nothing(monkeypatch):
    """mixup_prob 0: the draw says no mix, so the step runs the plain im2col and the hard loss."""
    calls = []
    real_ce = torch_ops.cross_entropy
    monkeypatch.setattr(torch_ops, "cross_entropy", lambda *a, **k: calls.append(tuple(k)) or real_ce(*a, **k))
    m = FSDPViT(tiny_cfg(mixup=0.8, mixup_prob=0.0), dtype=torch.float32, seed=3)
    ref = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    images, target = torch.randn(4, 3, 32, 32), torch.tensor([1, 5, 7, 2])
    assert m.forward_backward(images, target).item() == ref.forward_backward(images, target).item()
    assert calls == [("want_grad",), ("want_grad",)]


def test_eval_never_mixes():
    a = FSDPViT(tiny_cfg(**DEIT), dtype=torch.float32, seed=3).eval()
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3).eval()
    images = torch.randn(4, 3, 32, 32)
    assert torch.equal(a(images), b(images))


def test_resume_draws_what_an_uninterrupted_run_draws(tmp_path):
    opts = dict(model=DEIT, steps=4, global_batch=8)
    full = launch(1, opts, str(tmp_path / "a.json"))
    path = str(tmp_path / "ck_{rank}.pt")
    launch(1, dict(opts, save_at=2, save_path=path), str(tmp_path / "b.json"))
    resumed = launch(1, dict(opts, resume_from=path, resume_step=2), str(tmp_path / "c.json"))
    assert resumed["losses"] == pytest.approx(full["losses"][2:], rel=1e-6, abs=1e-7)
    plain = launch(1, dict(steps=4, global_batch=8), str(tmp_path / "d.json"))
    assert any(abs(a - b) > 1e-3 for a, b in zip(plain["losses"], full["losses"]))


def test_two_ranks_each_use_their_own_draw(tmp_path):
    """W = 2 on gloo: the first step's loss is the mean of each rank's loss on its own half-batch mixed with its own
    draw, and the gradient is the mean of those gradients (compared through its norm)."""
    cfg = tiny_cfg(**DEIT)
    res = launch(2, dict(model=DEIT, steps=1, global_batch=8), str(tmp_path / "r.json"))
    g = torch.Generator().manual_seed(1234)  # the batches dist_worker draws
    images = torch.randn(8, 8, 3, cfg.image_size, cfg.image_size, generator=g)
    targets = torch.randint(0, cfg.num_classes, (8, 8), generator=g)
    draws = [vit.draw_mix(cfg, vit.mix_rng(0, 0, r)) for r in (0, 1)]
    assert draws[0] != draws[1]
    losses, grads = [], []
    for r in (0, 1):
        model = FSDPViT(cfg, dtype=torch.float32, seed=0)
        model.rank = r  # the rank only selects the mixing draw (and stochastic-depth offsets) here
        losses.append(model.forward_backward(images[0, 4 * r:4 * r + 4], targets[0, 4 * r:4 * r + 4]).item())
        grads.append(full_grads_of(model))
    assert res["losses"][0] == pytest.approx(sum(losses) / 2, rel=1e-5)
    norm = sum(((grads[0][k] + grads[1][k]) / 2).double().pow(2).sum() for k in grads[0]).sqrt().item()
    assert res["norms"][0] == pytest.approx(norm, rel=1e-4)
    # with rank 0's draw on both halves the result would be another one
    swapped = FSDPViT(cfg, dtype=torch.float32, seed=0)
    l1_with_rank0_draw = swapped.forward_backward(images[0, 4:8], targets[0, 4:8]).item()
    assert abs(l1_with_rank0_draw - losses[1]) > 1e-4


# ------------------------------------------------------------------------------------------------
# flags, refusals
# ------------------------------------------------------------------------------------------------
def test_cli_parsing_and_config():
    a = parse_args([])
    assert (a.mixup, a.cutmix, a.mixup_prob, a.mixup_switch_prob, a.smoothing) == (0.0, 0.0, 1.0, 0.5, 0.0)
    assert not ViTConfig.from_args(a).mixing
    a = parse_args(["--mixup", "0.8", "--cutmix", "1.0", "--smoothing", "0.1", "--mixup_prob", "0.5",
                    "--mixup_switch_prob", "0.25"])
    c = ViTConfig.from_args(a)
    assert (c.mixup, c.cutmix, c.smoothing, c.mixup_prob, c.mixup_switch_prob) == (0.8, 1.0, 0.1, 0.5, 0.25)
    assert c.mixing and ViTConfig(cutmix=0.5).mixing


@pytest.mark.parametrize("flag,bad", [("--mixup", "-0.1"), ("--mixup", "nan"), ("--cutmix", "inf"),
                                      ("--mixup_prob", "1.5"), ("--mixup_prob", "-1"), ("--mixup_switch_prob", "2"),
                                      ("--smoothing", "1"), ("--smoothing", "-0.1"), ("--smoothing", "nan")])
def test_cli_rejects_invalid_values(flag, bad):
    with pytest.raises(SystemExit):
        parse_args([flag, bad])
    with pytest.raises(ValueError):
        ViTConfig(**{flag[2:]: float(bad)})


def test_odd_local_batch_is_refused():
    model = FSDPViT(tiny_cfg(cutmix=1.0), dtype=torch.float32, seed=3)
    with pytest.raises(ValueError, match="even local batch"):
        model.forward_backward(torch.randn(3, 3, 32, 32), torch.tensor([1, 2, 3]))
    # smoothing alone pairs nothing: an odd batch is fine
    FSDPViT(tiny_cfg(smoothing=0.1), dtype=torch.float32, seed=3).forward_backward(torch.randn(3, 3, 32, 32),
                                                                                  torch.tensor([1, 2, 3]))


def test_cli_refuses_an_odd_local_batch_at_start_up(tmp_path):
    args = ["--fake_data", "--device", "cpu", "--nproc", "2", "--image_size", "32", "--patch_size", "8", "--embed_dim",
            "32", "--num_heads", "2", "--num_blocks", "1", "--num_classes", "10", "--batch_size", "6", "--max_steps",
            "1", "--num_workers", "0", "--mixup", "0.8", "--ckpt_dir", str(tmp_path)]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "run_vit_training.py", *args], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode != 0
    assert "even local batch" in r.stdout + r.stderr and "training begins" not in r.stdout


def test_cuda_graph_refuses_mixing_and_accepts_smoothing():
    for kw in (dict(mixup=0.8), dict(cutmix=1.0)):
        model = FSDPViT(tiny_cfg(**kw), dtype=torch.float32, seed=3)
        with pytest.raises(RuntimeError, match="mixup / cutmix"):
            GraphedTrainStep(model, ShardedAdamW(model, lr=1e-3))
    model = FSDPViT(tiny_cfg(smoothing=0.1), dtype=torch.float32, seed=3)
    with pytest.raises(RuntimeError, match="CUDA model"):  # gets past the mixing check; CPU models have no graphs
        GraphedTrainStep(model, ShardedAdamW(model, lr=1e-3))


# ------------------------------------------------------------------------------------------------
# build: the changed kernels stay spill-free
# ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")),
                    reason="needs nvcc")
def test_im2col_and_cross_entropy_compile_for_sm90a_without_spills(tmp_path):
    from vit_10b_fsdp_example_b200 import build_ext

    nvcc = os.path.join(build_ext._cuda_home(), "bin", "nvcc")
    res = subprocess.run([nvcc, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, "elementwise.cu"), "-o", str(tmp_path / "e.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = (res.stdout + res.stderr).splitlines()
    found = {}
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln and ("im2col_kernel" in ln or "cross_entropy_kernel" in ln):
            assert "sm_90a" in ln
            spill = next(x for x in lines[i + 1:] if "spill stores" in x)
            found[ln.split("'")[1]] = spill
    assert sum("im2col_kernel" in k for k in found) == 6  # fp32 / bf16 images x no mix / Mixup / CutMix
    assert sum("cross_entropy_kernel" in k for k in found) == 1
    assert all("0 bytes spill stores, 0 bytes spill loads" in v for v in found.values()), found
