"""QK normalisation on the GPU: the qk_norm kernels against fp64 references computed from the same bf16 inputs, their
argument checks, and the model with --qk_norm against the fp32 CPU model, across activation-keeping modes, under CUDA
graphs and through the command line.

Tolerances are derived from the kernels' arithmetic and written beside each check: a bf16 output is rounded once
(half an ulp, 2^-9 relative; one ulp, 2^-8, is allowed), and the fp32 statistics are off from fp64 by a few fp32 ulps of
the quantities they are computed from."""
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
BF16_ULP = 2.0 ** -8
F32_EPS = 2.0 ** -23
HEAD_DIMS = [32, 40, 48, 56, 64, 72, 80, 88, 96, 104, 112, 120, 128, 136, 144, 152, 160, 256]
SHAPES = [(37, 1), (513, 3), (1031, 16), (257, 32)]  # (T, H): T odd and not a multiple of any tile


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _inputs(T, H, hd, seed):
    """bf16 qkv [T, 3D] with constant rows and rows whose |mean| >> std, and weights with zero entries."""
    g = torch.Generator().manual_seed(seed)
    D = H * hd
    x = torch.randn(T, 3 * D, generator=g) * 2 + torch.randn(T, 1, generator=g)
    x = x.view(T, 3, H, hd)
    x[::7, 0, 0] = 1.5                                        # constant q rows
    x[3::11, 1, H - 1] = -0.75                                # constant k rows
    x[5::13, 0] = 200.0 + torch.randn(x[5::13, 0].shape, generator=g) * 0.5   # |mean| >> std
    x[2::9, 1] = -50.0 + torch.randn(x[2::9, 1].shape, generator=g) * 0.1
    w = [torch.randn(hd, generator=g) * 0.5 + 1.0, torch.randn(hd, generator=g) * 0.2,
         torch.randn(hd, generator=g) * 0.5 + 1.0, torch.randn(hd, generator=g) * 0.2]
    w[0][::5] = 0.0                                           # zero-gamma entries
    w[2][1::6] = 0.0
    return x.view(T, 3 * D).to(torch.bfloat16), [t.to(torch.bfloat16) for t in w]


def _ref_fwd(qkv, H, hd, w, eps=1e-5):
    """fp64 LayerNorm of the q / k heads of the bf16 input: (y [T, 2, H, hd], mean, rstd [T, 2, H], xhat)."""
    T = qkv.shape[0]
    x = qkv.double()[:, : 2 * H * hd].view(T, 2, H, hd)
    mean = x.mean(-1)
    rstd = torch.rsqrt(x.var(-1, unbiased=False) + eps)
    xhat = (x - mean[..., None]) * rstd[..., None]
    gamma = torch.stack([w[0].double(), w[2].double()])[None, :, None, :]
    beta = torch.stack([w[1].double(), w[3].double()])[None, :, None, :]
    return xhat * gamma + beta, mean, rstd, xhat, gamma


def _check(what, got, ref, tol):
    got = got.double()
    bad = (got - ref).abs() > tol
    if bad.any():
        i = (((got - ref).abs() - tol) / (tol + 1e-30)).flatten().argmax().item()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside tolerance; worst got "
                             f"{got.flatten()[i].item():.7g} ref {ref.flatten()[i].item():.7g} "
                             f"tol {tol.flatten()[i].item():.3g}")


def _fwd_and_check(T, H, hd, inplace, ld_pad, seed):
    co = _co()
    D = H * hd
    qkv_c, w_c = _inputs(T, H, hd, seed)
    ld = 3 * D + ld_pad
    buf = torch.full((T, ld), float("nan"), dtype=torch.bfloat16, device="cuda")  # padding a kernel must not read
    qkv = buf[:, : 3 * D]
    qkv.copy_(qkv_c.cuda())
    if inplace:
        qkv[:, 2 * D:] = float("nan")  # sentinel: an in-place kernel writing past column 2D or reading v fails
    w = [t.cuda() for t in w_c]
    out, mean, rstd = co.qk_norm_fwd(qkv, H, hd, *w, 1e-5, inplace=inplace)
    torch.cuda.synchronize()
    y, m, r, xhat, gamma = _ref_fwd(qkv_c, H, hd, w_c)
    # statistics: mean is an fp32 sum of hd bf16 values (error <= hd * eps32 * mean|x|); rstd from the two-pass fp32
    # variance, off by a few eps32 relative plus the mean's error squared into the variance (|mean| >> std rows)
    absx = qkv_c.double()[:, : 2 * D].view(T, 2, H, hd).abs()
    _check("mean", mean.cpu().view(T, 2, H), m, hd * F32_EPS * absx.mean(-1) + 1e-30)
    mean_err = hd * F32_EPS * absx.mean(-1)
    _check("rstd", rstd.cpu().view(T, 2, H), r, r * (16 * F32_EPS + 2 * (mean_err * r) ** 2 + 4 * hd * F32_EPS))
    # output: one bf16 rounding (<= 1 ulp of |ref|) plus |gamma| times the error of xhat in fp32, which is that of the
    # statistics: (mean error + eps32 |x|) * rstd + |xhat| * rel. error of rstd
    ex = (mean_err[..., None] + 4 * F32_EPS * absx) * r[..., None] + xhat.abs() * 32 * hd * F32_EPS
    got = out.cpu()[:, : 2 * D].view(T, 2, H, hd)
    _check("qk_norm_fwd out", got, y, BF16_ULP * y.abs() + gamma.abs() * ex + 1e-6)
    if inplace:
        assert out.data_ptr() == qkv.data_ptr()
        assert torch.isnan(buf[:, 2 * D:].float()).all(), "the in-place forward touched the v columns or the padding"
    else:
        assert torch.equal(out[:, 2 * D:].cpu(), qkv_c[:, 2 * D:]), "v was not copied bit for bit"
        assert torch.isnan(buf[:, 3 * D:].float()).all()
    return qkv, qkv_c, w, w_c, mean, rstd


@pytest.mark.parametrize("inplace", [True, False])
@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_kernels_against_fp64(hd, inplace):
    i = HEAD_DIMS.index(hd)
    T, H = SHAPES[(i + int(inplace)) % len(SHAPES)]
    D = H * hd
    ld_pad = 8 if i % 2 else 0
    qkv, qkv_c, w, w_c, mean, rstd = _fwd_and_check(T, H, hd, inplace, ld_pad, seed=hd * 10 + int(inplace))
    if inplace:  # the backward reads the un-normalised values
        qkv = torch.empty(T, 3 * D + ld_pad, dtype=torch.bfloat16, device="cuda")[:, : 3 * D]
        qkv.copy_(qkv_c.cuda())
    # backward
    g = torch.Generator().manual_seed(hd)
    dy_c = (torch.randn(T, 3 * D, generator=g) * torch.rand(T, 1, generator=g) * 4).to(torch.bfloat16)
    dqkv = dy_c.cuda()
    _, dwq, dbq, dwk, dbk, cs = _co().qk_norm_bwd(dqkv, qkv, H, hd, w[0], w[2], mean, rstd)
    torch.cuda.synchronize()
    _, m, r, xhat, gamma = _ref_fwd(qkv_c, H, hd, w_c)
    dy = dy_c.double()[:, : 2 * D].view(T, 2, H, hd)
    gy = dy * gamma
    s1 = gy.mean(-1, keepdim=True)
    s2 = (gy * xhat).mean(-1, keepdim=True)
    dx = r[..., None] * (gy - s1 - xhat * s2)
    # dx: one bf16 rounding, plus the fp32 error of r * (gy - s1 - xhat s2): the terms' magnitudes times a few hd eps32,
    # and the error of xhat (from the fp32 statistics) times |s2|, all times rstd (up to 1 / sqrt(eps) on constant rows)
    absx = qkv_c.double()[:, : 2 * D].view(T, 2, H, hd).abs()
    mean_err = hd * F32_EPS * absx.mean(-1, keepdim=True)
    ex = (mean_err + 4 * F32_EPS * absx) * r[..., None] + xhat.abs() * 32 * hd * F32_EPS
    terms = gy.abs() + s1.abs() + (xhat.abs() + ex) * s2.abs()
    tol = BF16_ULP * dx.abs() + r[..., None] * (8 * hd * F32_EPS * terms + ex * s2.abs()) + 1e-6
    got = dqkv.cpu()
    _check("qk_norm_bwd dx", got[:, : 2 * D].view(T, 2, H, hd), dx, tol)
    assert torch.equal(got[:, 2 * D:], dy_c[:, 2 * D:]), "dv changed"
    # dw / db: fp32 sums over T * H rows: 1e-5 of the sum of the terms' magnitudes (reordered fp32 additions), plus the
    # xhat error of each term for dw
    for side, (dw_, db_) in enumerate(((dwq, dbq), (dwk, dbk))):
        d, xh, e = dy[:, side], xhat[:, side], ex[:, side]
        _check(f"dw[{side}]", dw_.cpu(), (d * xh).sum((0, 1)), 1e-5 * (d * xh).abs().sum((0, 1)) + (d.abs() * e).sum((0, 1)) + 1e-6)
        _check(f"db[{side}]", db_.cpu(), d.sum((0, 1)), 1e-5 * d.abs().sum((0, 1)) + 1e-6)
    # column sums of the stored bf16 dq / dk: exact inputs, fp32 accumulation -> 1e-6 of the sum of magnitudes
    stored = got[:, : 2 * D].double()
    _check("colsum", cs.cpu(), stored.sum(0), 1e-6 * stored.abs().sum(0) + 1e-6)


@pytest.mark.parametrize("T,H", SHAPES + [(1, 1), (2, 16)])
def test_every_shape_at_hd_64_and_160(T, H):
    for hd in (64, 160):
        for inplace in (True, False):
            _fwd_and_check(T, H, hd, inplace, 0, seed=T + H + hd)


def test_rejects_bad_head_dims_and_leading_dims():
    co = _co()
    w = [torch.ones(12, dtype=torch.bfloat16, device="cuda") for _ in range(4)]
    qkv = torch.zeros(4, 3 * 12, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match=r"hd % 8 == 0 and 8 <= hd <= 256"):
        co.qk_norm_fwd(qkv, 1, 12, *w, 1e-5)
    w = [torch.ones(264, dtype=torch.bfloat16, device="cuda") for _ in range(4)]
    qkv = torch.zeros(4, 3 * 264, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match=r"hd % 8 == 0 and 8 <= hd <= 256"):
        co.qk_norm_fwd(qkv, 1, 264, *w, 1e-5)
    w = [torch.ones(64, dtype=torch.bfloat16, device="cuda") for _ in range(4)]
    bad = torch.zeros(4, 3 * 128 + 4, dtype=torch.bfloat16, device="cuda")[:, : 3 * 128]  # ld = 388: 776 bytes
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        co.qk_norm_fwd(bad, 2, 64, *w, 1e-5)
    good = torch.zeros(4, 3 * 128, dtype=torch.bfloat16, device="cuda")
    _, mean, rstd = co.qk_norm_fwd(good, 2, 64, *w, 1e-5)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        co.qk_norm_bwd(bad, good, 2, 64, w[0], w[2], mean, rstd)


# ------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=3, mlp_ratio=4.0, num_classes=96,
             qk_norm=True)
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


def _randomize_norms(model, seed=0):
    from helpers import full_params_of

    g = torch.Generator().manual_seed(seed)
    full = {k: v.cpu() for k, v in full_params_of(model).items()}
    for k, v in full.items():
        if "_norm." in k:
            full[k] = (1.0 if k.endswith("weight") else 0.0) + 0.5 * torch.randn(v.shape, generator=g)
    model.load_full_state_dict(full)


@pytest.mark.parametrize("route", ["fused", "unfused"])
def test_model_matches_the_fp32_cpu_model(route):
    """Same parameters (host init, random norm weights): bf16 GPU vs fp32 CPU loss and gradients.  fused: N = 256,
    hd 64 (the wgmma attention kernels); unfused: N = 225 (odd) and hd 80 (GEMM + softmax route)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg() if route == "fused" else _cfg(image_size=210, embed_dim=320)
    assert cuda_ops.use_flash(cfg.num_patches, cfg.head_dim) == (route == "fused")
    x, y = _data(cfg)
    for keep in (0, 3):
        res = []
        for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
            model = FSDPViT(cfg, device=dev, dtype=dtype, seed=4, ckpt_keep_blocks=keep)
            _randomize_norms(model)
            loss = model.forward_backward(x.to(dev), y.to(dev)).item()
            res.append((loss, _named_grads(model)))
        (loss_ref, g_ref), (loss, grads) = res
        assert math.isfinite(loss) and abs(loss - loss_ref) < 1e-2 * abs(loss_ref) + 1e-2, (keep, loss, loss_ref)
        assert any("q_norm" in k for k in g_ref)
        for k in g_ref:
            a, b = g_ref[k], grads[k]
            if k.endswith("k_norm.bias"):  # zero in exact arithmetic (the softmax cancels q . b_k): rounding only
                assert b.abs().max().item() <= 1e-2 * grads[k.replace("bias", "weight")].abs().max().item() + 1e-6
                continue
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (keep, k)
    # the norm matters: without it the loss is another one
    ref0 = FSDPViT(_cfg(qk_norm=False) if route == "fused" else _cfg(image_size=210, embed_dim=320, qk_norm=False),
                   device="cuda", dtype=torch.bfloat16, seed=4)
    assert abs(ref0.forward_backward(x.cuda(), y.cuda()).item() - loss) > 1e-3


@pytest.mark.parametrize("kw", [dict(), dict(embed_dim=320, image_size=210), dict(att_dropout=0.1, mlp_dropout=0.1)])
def test_checkpointed_kept_and_uncheckpointed_blocks_give_the_same_gradients(kw):
    """GEMM-produced weight gradients are bitwise equal; biases, LayerNorm and QK-norm parameters are reduced with fp32
    atomics in arrival order, whose last bits vary from run to run: one bf16 ulp."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg(**kw)
    x, y = _data(cfg)
    runs = []
    for mkw in (dict(grad_ckpt=True, ckpt_keep_blocks=0), dict(grad_ckpt=True, ckpt_keep_blocks=3),
                dict(grad_ckpt=False)):
        model = FSDPViT(cfg, device="cuda", dtype=torch.bfloat16, seed=4, **mkw)
        if mkw.get("ckpt_keep_blocks") == 3:
            model.keep_extras = {"P": 1, "h": 2, "g": 3}
        _randomize_norms(model)
        runs.append((model.forward_backward(x.cuda(), y.cuda()).item(), _named_grads(model)))
    (l0, g0) = runs[0]
    for l1, g1 in runs[1:]:
        assert abs(l0 - l1) <= 1e-6 * abs(l0), (l0, l1)
        for k in g0:
            linear_weight = k.endswith(("qkv.weight", "proj.weight", "fc1.weight", "fc2.weight", "head.weight"))
            diff = (g0[k] - g1[k]).abs().max().item()
            if linear_weight:
                assert torch.equal(g0[k], g1[k]), (k, diff, g0[k].abs().max().item())
            elif k.endswith("k_norm.bias"):
                # zero in exact arithmetic (the softmax cancels q . b_k): each entry is the rounding left by a sum of
                # cancelling terms, so two arrival orders differ on the scale of the largest entry, not of each entry
                assert diff <= 2.0 ** -7 * g0[k].abs().max().item() + 1e-12, (k, diff, g0[k].abs().max().item())
            else:
                one_ulp = g0[k].abs() * 2.0 ** -7 + 1e-6 * g0[k].abs().max().item()  # bf16: 8 significant bits
                assert ((g0[k] - g1[k]).abs() <= one_ulp).all(), (k, diff, g0[k].abs().max().item())


def test_cuda_graph_matches_eager():
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

    cfg = _cfg(image_size=112, embed_dim=320, num_heads=2)
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


def test_cli_trains_with_qk_norm(tmp_path):
    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "16",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--num_epochs", "1", "--ckpt_epoch_interval", "100", "--test_epoch_interval", "100", "--qk_norm"]
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(tmp_path / "ckpt")], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "qk_norm=True" in r.stdout
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
