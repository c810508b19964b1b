"""Rotary position embedding on the GPU: rope_fwd / rope_bwd and the RoPE-fused qk_norm kernels against fp64 references
computed from the same bf16 inputs, their argument checks, and the model with --rope against the fp32 CPU model on
both attention routes, across activation-keeping modes, under CUDA graphs and through the command line.

Tolerances are derived beside each check.  A bf16 output is rounded once (2^-9 relative; one ulp, 2^-8, is allowed).
The fp32 tables are off from the fp64 closed form by half an fp32 ulp (2^-24) of |cos| and |sin| <= 1, which moves
y0 = x0 c - x1 s by at most 2^-24 (|x0| + |x1|); the fp32 products and sum add a few more ulps of the same size, so
2^-21 (|x0| + |x1|) bounds everything but the final rounding."""
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
HEAD_DIMS = [32, 40, 48, 56, 64, 72, 80, 88, 96, 104, 112, 120, 128, 136, 144, 152, 160, 256]  # test_gpu_qk_norm's
CASES = [(3, 0, False), (2, 1, True), (5, 5, False), (4, 5, True), (3, 1, False)]  # (B, P, with keep)
GRID = 7  # N = 49 patches: T = P + 49 or P + 23 kept, odd at P in {0, 1}


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _tables(hd, grid=GRID):
    from vit_10b_fsdp_example_b200.models import vit

    cos, sin = vit.rope_tables(grid, hd, 10000.0)
    F_ = hd // 4
    n = torch.arange(grid * grid, dtype=torch.float64)
    w = 10000.0 ** (-torch.arange(F_, dtype=torch.float64) / F_)
    ang = torch.cat([(n // grid)[:, None] * w, (n % grid)[:, None] * w], dim=1)  # the closed form in fp64
    return cos.cuda(), sin.cuda(), ang


def _keep(B, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randperm(N, generator=g)[:K].sort()[0] for _ in range(B)]).int()


def _rows(B, T, P, keep):
    """Table row of every token row (-1 for prefix rows)."""
    idx = torch.full((B, T), -1, dtype=torch.long)
    idx[:, P:] = keep.long() if keep is not None else torch.arange(T - P)
    return idx.reshape(-1)


def _rot64(x, ang, rows, transpose=False):
    """fp64 R x (or R^T x) on [rows, W] with pairs interleaved; rows with table row -1 are copied."""
    y = x.double().clone()
    m = rows >= 0
    half = ang.shape[1]
    xp = y[m].view(int(m.sum()), -1, half, 2)
    c, s = torch.cos(ang[rows[m]])[:, None], torch.sin(ang[rows[m]])[:, None]
    if transpose:
        s = -s
    x0, x1 = xp[..., 0], xp[..., 1]
    y[m] = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), -1).view(int(m.sum()), -1)
    return y


def _pair_abs(x):
    """|x0| + |x1| of every pair, at both elements of the pair."""
    a = x.double().abs().view(x.shape[0], -1, 2).sum(-1, keepdim=True)
    return a.expand(-1, -1, 2).reshape(x.shape)


def _padded(T, width, pad, seed, scale=2.0):
    """bf16 [T, width] view of a [T, width + pad] buffer whose padding is NaN (it must stay untouched)."""
    g = torch.Generator().manual_seed(seed)
    buf = torch.full((T, width + pad), float("nan"), dtype=torch.bfloat16)
    buf[:, :width] = (torch.randn(T, width, generator=g) * scale).bfloat16()
    return buf.cuda()[:, :width]


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_rope_kernels_against_fp64(hd):
    co = _co()
    cos, sin, ang = _tables(hd)
    N = GRID * GRID
    for ci, (B, P, with_keep) in enumerate(CASES):
        H = 1 + (hd + ci) % 3
        D = H * hd
        K = 23 if with_keep else N
        keep = _keep(B, N, K, hd + ci).cuda() if with_keep else None
        T = P + K
        rows = _rows(B, T, P, keep.cpu() if keep is not None else None)
        pad = 8 * (ci % 2)
        x = _padded(B * T, 3 * D, pad, seed=hd * 31 + ci)
        xc = x.cpu()
        ref = _rot64(xc[:, : 2 * D], ang, rows)
        tol = BF16_ULP * ref.abs() + 2.0 ** -21 * _pair_abs(xc[:, : 2 * D])
        for inplace in (False, True):
            xi = x if not inplace else _padded(B * T, 3 * D, pad, seed=hd * 31 + ci)
            out = co.rope_fwd(xi, H, hd, cos, sin, B, P, keep, inplace=inplace)
            oc = out.cpu()
            assert ((oc[:, : 2 * D].double() - ref).abs() <= tol).all(), (hd, ci, inplace)
            assert torch.equal(oc[:, 2 * D:], xc[:, 2 * D:])  # v, bit for bit
            pre = rows < 0
            assert torch.equal(oc[pre], xc[pre])  # prefix rows, bit for bit
            if inplace and pad:
                assert torch.isnan(xi.as_strided((B * T, pad), (xi.stride(0), 1), 3 * D).cpu()).all()
        # backward: R^T in place, dv untouched, colsum of the stored values
        dy = _padded(B * T, 3 * D, pad, seed=hd * 37 + ci)
        dyc = dy.cpu()
        ref = _rot64(dyc[:, : 2 * D], ang, rows, transpose=True)
        tol = BF16_ULP * ref.abs() + 2.0 ** -21 * _pair_abs(dyc[:, : 2 * D])
        _, cs = co.rope_bwd(dy, H, hd, cos, sin, B, P, keep)
        dc = dy.cpu()
        assert ((dc[:, : 2 * D].double() - ref).abs() <= tol).all(), (hd, ci)
        assert torch.equal(dc[:, 2 * D:], dyc[:, 2 * D:]) and torch.equal(dc[rows < 0], dyc[rows < 0])
        if pad:
            assert torch.isnan(dy.as_strided((B * T, pad), (dy.stride(0), 1), 3 * D).cpu()).all()
        # fp32 sums of B * T bf16 values, in any order: B * T * 2^-24 of the sum of magnitudes
        want = dc[:, : 2 * D].double().sum(0)
        bound = B * T * 2.0 ** -23 * dc[:, : 2 * D].double().abs().sum(0) + 1e-30
        assert ((cs.cpu().double() - want).abs() <= bound).all()


def _ln64(x, w, b, eps=1e-5):
    m = x.mean(-1, keepdim=True)
    v = x.var(-1, unbiased=False, keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * w + b


@pytest.mark.parametrize("hd", HEAD_DIMS)
def test_fused_qk_norm_kernels_against_fp64(hd):
    co = _co()
    cos, sin, ang = _tables(hd)
    N = GRID * GRID
    for ci, (B, P, with_keep) in enumerate(CASES[:3]):
        H = 1 + (hd + ci) % 3
        D = H * hd
        K = 23 if with_keep else N
        keep = _keep(B, N, K, hd + ci).cuda() if with_keep else None
        T = P + K
        rows = _rows(B, T, P, keep.cpu() if keep is not None else None)
        pad = 8 * (ci % 2)
        g = torch.Generator().manual_seed(hd + ci)
        wq, bq, wk, bk = [(1.0 * (i % 2 == 0) + 0.5 * torch.randn(hd, generator=g)).bfloat16() for i in range(4)]
        w = [t.cuda() for t in (wq, bq, wk, bk)]
        x = _padded(B * T, 3 * D, pad, seed=hd * 41 + ci)
        xc = x.cpu().double()
        xq = xc[:, : 2 * D].view(B * T, 2, H, hd)
        yhat = torch.stack([_ln64(xq[:, 0], wq.double(), bq.double()), _ln64(xq[:, 1], wk.double(), bk.double())], 1)
        yhat = yhat.reshape(B * T, 2 * D)
        ref = _rot64(yhat, ang, rows)
        # one rounding, the table term, and the fp32 statistics: mean / rstd are off by a few fp32 ulps of the row's
        # scale, which moves each normalised value by about 2^-20 of |xhat w| <= the pair magnitudes of yhat + |b|
        tol = BF16_ULP * ref.abs() + 2.0 ** -18 * (_pair_abs(yhat) + 1.0)
        for inplace in (False, True):
            xi = x if not inplace else _padded(B * T, 3 * D, pad, seed=hd * 41 + ci)
            out, mean, rstd = co.qk_norm_fwd(xi, H, hd, *w, 1e-5, inplace=inplace, rope=(cos, sin, B, P, keep))
            oc = out.cpu()
            assert ((oc[:, : 2 * D].double() - ref).abs() <= tol).all(), (hd, ci, inplace)
            assert torch.equal(oc[:, 2 * D:], x.cpu()[:, 2 * D:])
        # backward: fp64 LayerNorm backward of R^T dy
        dy = _padded(B * T, 3 * D, pad, seed=hd * 43 + ci, scale=1.0)
        dyc = dy.cpu()
        xr = xc[:, : 2 * D].clone().requires_grad_(True)
        xv = xr.view(B * T, 2, H, hd)
        wd = [t.double().requires_grad_(True) for t in (wq, bq, wk, bk)]
        y = torch.stack([_ln64(xv[:, 0], wd[0], wd[1]), _ln64(xv[:, 1], wd[2], wd[3])], 1).reshape(B * T, 2 * D)
        y.backward(_rot64(dyc[:, : 2 * D], ang, rows, transpose=True))
        _, dwq, dbq, dwk, dbk, cs = co.qk_norm_bwd(dy, x, H, hd, w[0], w[2], mean, rstd, rope=(cos, sin, B, P, keep))
        dx = dy.cpu()[:, : 2 * D].double()
        # dx = rstd (dy w - s1 - xhat s2): fp32 sums over hd terms cancel, so the error is on the scale of the row's
        # largest term, rstd |dy w|, times a few hd fp32 ulps; plus the one rounding
        wmax = max(wq.float().abs().max().item(), wk.float().abs().max().item())
        scale = dyc[:, : 2 * D].double().abs().view(B * T, 2 * H, hd).amax(-1, keepdim=True) * wmax
        scale = (scale * rstd.cpu().double().view(B * T, 2 * H, 1)).expand(-1, -1, hd).reshape(B * T, 2 * D)
        tol = BF16_ULP * xr.grad.abs() + hd * 2.0 ** -20 * scale
        assert ((dx - xr.grad).abs() <= tol).all(), (hd, ci)
        assert torch.equal(dy.cpu()[:, 2 * D:], dyc[:, 2 * D:])
        for got, ref_g in ((dwq, wd[0].grad), (dbq, wd[1].grad), (dwk, wd[2].grad), (dbk, wd[3].grad)):
            assert (got.cpu().double() - ref_g).norm() <= 1e-2 * ref_g.norm() + 1e-6
        want = dx.sum(0)
        bound = B * T * 2.0 ** -23 * dx.abs().sum(0) + 1e-30  # column sums of the stored values, fp32 in any order
        assert ((cs.cpu().double() - want).abs() <= bound).all()


def test_rejects_bad_arguments_with_the_check_named():
    co = _co()
    cos, sin, _ = _tables(64)
    qkv = torch.zeros(2 * 49, 3 * 128, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match=r"hd % 8 == 0 and 8 <= hd <= 256"):
        c12, s12 = torch.zeros(49, 6, device="cuda"), torch.zeros(49, 6, device="cuda")
        co.rope_fwd(torch.zeros(98, 36, dtype=torch.bfloat16, device="cuda"), 1, 12, c12, s12, 2, 0)
    with pytest.raises(RuntimeError, match=r"hd % 8 == 0 and 8 <= hd <= 256"):
        c, s = torch.zeros(49, 132, device="cuda"), torch.zeros(49, 132, device="cuda")
        co.rope_fwd(torch.zeros(98, 3 * 264, dtype=torch.bfloat16, device="cuda"), 1, 264, c, s, 2, 0)
    bad = torch.zeros(98, 3 * 128 + 4, dtype=torch.bfloat16, device="cuda")[:, : 3 * 128]  # ld 388: 776 bytes
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        co.rope_fwd(bad, 2, 64, cos, sin, 2, 0)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        co.rope_bwd(bad, 2, 64, cos, sin, 2, 0)
    with pytest.raises(RuntimeError, match="expected a bf16 tensor"):
        co.rope_fwd(qkv.half(), 2, 64, cos, sin, 2, 0)
    with pytest.raises(RuntimeError, match=r"cos / sin tables must be contiguous fp32 CUDA \[N, hd / 2\]"):
        co.rope_fwd(qkv, 2, 64, cos.double(), sin.double(), 2, 0)
    with pytest.raises(RuntimeError, match=r"cos / sin tables must be contiguous fp32 CUDA \[N, hd / 2\]"):
        co.rope_fwd(qkv, 2, 64, cos[:, :16].contiguous(), sin[:, :16].contiguous(), 2, 0)
    with pytest.raises(RuntimeError, match=r"table has 48 rows but every image has T - P = 49"):
        co.rope_fwd(qkv, 2, 64, cos[:48].contiguous(), sin[:48].contiguous(), 2, 0)
    with pytest.raises(RuntimeError, match="are not B = 3 images"):
        co.rope_fwd(qkv, 2, 64, cos, sin, 3, 0)
    keep = torch.zeros(2, 48, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match=r"keep must be \[B, T - P\] = \[2, 49\]"):
        co.rope_fwd(qkv, 2, 64, cos, sin, 2, 0, keep)
    with pytest.raises(RuntimeError, match="keep must be a contiguous int32 CUDA tensor"):
        co.rope_fwd(qkv, 2, 64, cos, sin, 2, 0, torch.zeros(2, 49, dtype=torch.int64, device="cuda"))
    huge = torch.zeros(1, 3 * 128, dtype=torch.bfloat16, device="cuda").expand(2 ** 31, 3 * 128)
    with pytest.raises(RuntimeError, match="overflow 32 bits"):
        co.rope_fwd(huge, 2, 64, cos, sin, 1, 0, inplace=True)
    w = [torch.ones(64, dtype=torch.bfloat16, device="cuda") for _ in range(4)]
    with pytest.raises(RuntimeError, match=r"qk_norm_rope_fwd: table has 48 rows"):
        co.qk_norm_fwd(qkv, 2, 64, *w, 1e-5, rope=(cos[:48].contiguous(), sin[:48].contiguous(), 2, 0, None))
    _, mean, rstd = co.qk_norm_fwd(qkv, 2, 64, *w, 1e-5, rope=(cos, sin, 2, 0, None))
    with pytest.raises(RuntimeError, match="qk_norm_rope_bwd: .*are not B = 3 images"):
        co.qk_norm_bwd(qkv.clone(), qkv, 2, 64, w[0], w[2], mean, rstd, rope=(cos, sin, 3, 0, None))


# ------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=3, mlp_ratio=4.0, num_classes=96,
             rope=True)
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
    """Random norm and prefix parameters."""
    from helpers import full_params_of

    g = torch.Generator().manual_seed(seed)
    full = {k: v.cpu() for k, v in full_params_of(model).items()}
    for k, v in full.items():
        if "_norm." in k:
            full[k] = (1.0 if k.endswith("weight") else 0.0) + 0.5 * torch.randn(v.shape, generator=g)
        elif k in ("cls_token", "reg_token"):
            full[k] = torch.randn(v.shape, generator=g)
    model.load_full_state_dict(full)


ROUTES = {"fused": dict(), "unfused": dict(image_size=210, embed_dim=320, class_token=True, reg_tokens=1)}


def _gpu_vs_cpu(cfg, mode, x, y):
    """(loss error, {parameter: gradient error norm}, fp32 CPU gradients) of the bf16 GPU model against the fp32 CPU
    model from the same parameters."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    res = []
    for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
        model = FSDPViT(cfg, device=dev, dtype=dtype, seed=4, **mode)
        _randomize(model)
        loss = model.forward_backward(x.to(dev), y.to(dev)).item()
        res.append((loss, _named_grads(model)))
    (loss_ref, g_ref), (loss, grads) = res
    assert math.isfinite(loss)
    return abs(loss - loss_ref), {k: (g_ref[k] - grads[k]).norm().item() for k in g_ref}, g_ref


@pytest.mark.parametrize("route", ["fused", "unfused"])
@pytest.mark.parametrize("kw", [dict(), dict(qk_norm=True), dict(att_dropout=0.1), dict(patch_drop_rate=0.5),
                                dict(qk_norm=True, patch_drop_rate=0.5, att_dropout=0.1)])
def test_model_matches_the_fp32_cpu_model(route, kw):
    """bf16 GPU vs fp32 CPU loss and gradients, the qkv bias included, with every block checkpointed, kept, and not
    checkpointed.  fused: N = 256, hd 64 (the wgmma attention kernels); unfused: T = 227 (odd) tokens with a class and
    a register token, hd 80 (GEMM + softmax route).  The bf16 model's distance from the fp32 one is set by its bf16
    activations, not by the rotation: every gradient is held to 5 % of its norm, or to twice the distance the same
    model without --rope has from its fp32 twin (small gradients, such as norm1's, carry the rounding of the large
    activations they are reduced from)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    cfg = _cfg(**ROUTES[route], **kw)
    assert cuda_ops.use_flash(cfg.num_tokens, cfg.head_dim) == (route == "fused")
    x, y = _data(cfg)
    for mode in (dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=3), dict(grad_ckpt=False)):
        dloss, err, g_ref = _gpu_vs_cpu(cfg, mode, x, y)
        dloss0, err0, _ = _gpu_vs_cpu(_cfg(**ROUTES[route], **dict(kw, rope=False)), mode, x, y)
        assert dloss <= 1e-2 * abs(dloss0 + 1.0) + 2 * dloss0, (mode, dloss, dloss0)
        for k in g_ref:
            scale, rel = g_ref[k].norm().item(), 5e-2
            if k.endswith("k_norm.bias"):
                # without the rotation the softmax cancels q . b_k exactly; with it only the part that varies with the
                # position is left (about 15 % of the k_norm weight gradient here), a sum of cancelling terms whose
                # bf16 rounding does not cancel.  Measured on an H100: 12-19 % of the weight gradient's norm with
                # attention dropout, patch dropout and QK norm together; the fp32 CPU engine matches fp64 exactly there
                # (tests/test_rope.py), so the bound is the weight gradient's scale
                scale, rel = g_ref[k.replace("bias", "weight")].norm().item(), 0.25
            assert err[k] <= max(rel * scale, 2 * err0[k]) + 1e-6, (mode, k, err[k], err0[k], scale)
        D = cfg.embed_dim
        assert g_ref["blocks.0.attn.qkv.bias"][: 2 * D].norm() > 0


@pytest.mark.parametrize("qk_norm", [False, True])
def test_cuda_graph_matches_eager(qk_norm):
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

    cfg = _cfg(image_size=112, embed_dim=320, num_heads=2, qk_norm=qk_norm)
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
            assert len(model._rope_tables) == 1  # built once: the graph replays the same table pointers
    for a, b in zip(results["eager"], results["graph"]):
        assert abs(a - b) < 2e-2 * abs(a) + 1e-3, results


def test_cli_trains_with_rope(tmp_path):
    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "16",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--num_epochs", "1", "--ckpt_epoch_interval", "100", "--test_epoch_interval", "100", "--rope",
            "--rope_ref_grid", "16"]
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(tmp_path / "ckpt")], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "rope=True" in r.stdout
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
