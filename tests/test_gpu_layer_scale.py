"""LayerScale on the GPU: the layer_scale kernels against fp64 references computed from the same bf16 inputs, their
argument checks, and the model with --init_values against the fp32 CPU model, across activation-keeping modes, at
init_values 1 against the model without the flag, under CUDA graphs and through the command line.

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
F32_EPS = 2.0 ** -23
THREADS = 256  # threads per row in csrc/layer_scale.cu


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _gamma(D, g):
    """U(0.5, 1.5) with random signs, plus 1e-5, 1 and 0 entries."""
    sign = torch.where(torch.rand(D, generator=g) < 0.5, -1.0, 1.0)
    gamma = sign * (0.5 + torch.rand(D, generator=g))
    gamma[:: 7] = 1e-5
    gamma[3:: 11] = 1.0
    gamma[5:: 13] = 0.0
    return gamma


def _inputs(D, K, seed, dev="cuda"):
    g = torch.Generator().manual_seed(seed)
    W = (torch.randn(D, K, generator=g) * 0.02).bfloat16()
    b = (torch.randn(D, generator=g) * 0.02).bfloat16()
    gamma = _gamma(D, g).bfloat16()
    M = (torch.randn(D, K, generator=g) * torch.rand(D, 1, generator=g) * 5).bfloat16()
    S = torch.randn(D, generator=g) * 30
    return [t.to(dev) for t in (W, b, gamma, M, S)]


def _at_offset(t, off):
    """A copy of t that starts `off` elements into a flat buffer (so its rows are not 16-byte aligned)."""
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device=t.device)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    return v


def _check_kernels(W, b, gamma, M, S):
    """Fold and backward against the same fp32 products rounded on the host (bitwise) and dgamma against fp64."""
    co = _co()
    D, K = W.shape
    Wg, bg = co.layer_scale_fold(W, b, gamma)
    Mref = M.clone()
    dW = M  # overwritten in place: M in, gamma o M out
    Wg2, db, dgamma = co.layer_scale_bwd(W, b, gamma, dW, S)
    torch.cuda.synchronize()
    gf = gamma.float()
    # Wg, bg, dW: one fp32 product (relative error <= 2^-24) rounded once to bf16 -- the same operations torch runs, so
    # the results are bitwise equal; and within half a bf16 ulp of the exact product: bf16 keeps 8 significant bits, so
    # that is <= 2^-8 of |exact| (plus the fp32 product's 2^-24).
    want_wg = (W.float() * gf[:, None]).bfloat16()
    assert torch.equal(Wg, want_wg), (Wg.float() - want_wg.float()).abs().max()
    assert torch.equal(Wg2, Wg)
    assert torch.equal(bg, (b.float() * gf).bfloat16())
    assert torch.equal(dW, (Mref.float() * gf[:, None]).bfloat16())
    exact = W.double() * gamma.double()[:, None]
    assert ((Wg.double() - exact).abs() <= (2.0 ** -8 + 2.0 ** -23) * exact.abs()).all()
    # db = gamma * S: one fp32 product
    assert torch.equal(db, gf * S)
    # dgamma = sum_k W M + b S in fp32: each thread adds about K / 256 products in sequence (FMA), then a 5-level warp
    # tree and 8 warp partials, then b S: error <= (K / 256 + 16) eps32 * sum |W M| + 2 eps32 |b S|
    prod = W.double() * Mref.double()
    want = prod.sum(1) + b.double() * S.double()
    tol = (K / THREADS + 16) * F32_EPS * prod.abs().sum(1) + 2 * F32_EPS * (b.double() * S.double()).abs() + 1e-30
    err = (dgamma.double() - want).abs()
    assert (err <= tol).all(), f"dgamma: worst err {err.max().item():.3g}, tol there {tol[err.argmax()].item():.3g}"


@pytest.mark.parametrize("K", [5120, 20480])
def test_kernels_at_the_vit10b_shapes(K):
    _check_kernels(*_inputs(5120, K, seed=K))


@pytest.mark.parametrize("D,K", [(1, 1), (3, 7), (17, 13), (64, 8), (9, 24), (33, 1027), (5, 2047), (2, 4100)])
def test_kernels_at_small_and_odd_shapes(D, K):
    _check_kernels(*_inputs(D, K, seed=D * 7919 + K))


@pytest.mark.parametrize("offsets", [(3, 3), (0, 3), (1, 6)])
def test_kernels_on_unaligned_rows(offsets):
    """W and dW at odd offsets inside flat buffers (as the model's parameter and gradient views may be): their 16-byte
    phase differs from the freshly allocated Wg's, so every element takes the scalar path.  (With aligned bases and
    K % 8 != 0, as in the small-shape test, each row starts at another phase: scalar head, vector body, scalar tail.)"""
    W, b, gamma, M, S = _inputs(37, 1000, seed=sum(offsets))
    _check_kernels(_at_offset(W, offsets[0]), b, gamma, _at_offset(M, offsets[1]), S)


def test_rejects_bad_arguments():
    co = _co()
    W, b, gamma, M, S = _inputs(8, 16, seed=0)
    with pytest.raises(RuntimeError, match="layer_scale_fold: W must be a contiguous bf16 CUDA"):
        co.layer_scale_fold(W.float(), b, gamma)
    with pytest.raises(RuntimeError, match="layer_scale_fold: W must be a contiguous bf16 CUDA"):
        co.layer_scale_fold(W.t(), b, gamma)
    with pytest.raises(RuntimeError, match="b and gamma must be contiguous bf16 vectors of length D"):
        co.layer_scale_fold(W, b[:7], gamma)
    with pytest.raises(RuntimeError, match="b and gamma must be contiguous bf16 vectors of length D"):
        co.layer_scale_fold(W, b, gamma.float())
    with pytest.raises(RuntimeError, match="layer_scale_bwd: dW must be a contiguous bf16 matrix of W's shape"):
        co.layer_scale_bwd(W, b, gamma, M[:, :8], S)
    with pytest.raises(RuntimeError, match="S, db and dgamma must be contiguous fp32 vectors of length D"):
        co.layer_scale_bwd(W, b, gamma, M, S.bfloat16())
    with pytest.raises(RuntimeError, match="S, db and dgamma must be contiguous fp32 vectors of length D"):
        co.layer_scale_bwd(W, b, gamma, M, S[:4])


# ------------------------------------------------------------------------------------------------
# model level
# ------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=3, mlp_ratio=4.0, num_classes=96,
             init_values=1e-5)
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


def _randomize_gammas(model, seed=0):
    """U(0.5, 1.5) with mixed signs: at 1e-5 the branches barely move the loss and wrong gradients would pass."""
    from helpers import full_params_of

    g = torch.Generator().manual_seed(seed)
    full = {k: v.cpu() for k, v in full_params_of(model).items()}
    for k, v in full.items():
        if k.endswith(("ls1.gamma", "ls2.gamma")):
            sign = torch.where(torch.rand(v.shape, generator=g) < 0.5, -1.0, 1.0)
            full[k] = sign * (0.5 + torch.rand(v.shape, generator=g))
    model.load_full_state_dict(full)


@pytest.mark.parametrize("route", ["fused", "unfused"])
def test_model_matches_the_fp32_cpu_model(route):
    """Same parameters (host init, random gammas): bf16 GPU vs fp32 CPU loss and gradients.  fused: N = 256, hd 64
    (the wgmma attention kernels); unfused: N = 225 (odd) and hd 80 (GEMM + softmax route)."""
    from vit_10b_fsdp_example_b200.ops import cuda_ops
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg() if route == "fused" else _cfg(image_size=210, embed_dim=320)
    assert cuda_ops.use_flash(cfg.num_patches, cfg.head_dim) == (route == "fused")
    x, y = _data(cfg)
    for keep in (0, 3):
        res = []
        for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
            model = FSDPViT(cfg, device=dev, dtype=dtype, seed=4, ckpt_keep_blocks=keep)
            _randomize_gammas(model)
            loss = model.forward_backward(x.to(dev), y.to(dev)).item()
            res.append((loss, _named_grads(model)))
        (loss_ref, g_ref), (loss, grads) = res
        assert math.isfinite(loss) and abs(loss - loss_ref) < 1e-2 * abs(loss_ref) + 1e-2, (keep, loss, loss_ref)
        assert any(k.endswith("ls2.gamma") for k in g_ref)
        for k in g_ref:
            a, b = g_ref[k], grads[k]
            # bf16 activations and weights through three blocks: 5 % of the gradient's norm, as for --qk_norm
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (keep, k)


@pytest.mark.parametrize("kw", [dict(), dict(embed_dim=320, image_size=210), dict(att_dropout=0.1, mlp_dropout=0.1),
                                dict(drop_path_rate=0.5, qk_norm=True)])
def test_checkpointed_kept_and_uncheckpointed_blocks_give_the_same_gradients(kw):
    """GEMM-produced weight gradients (scaled by gamma in one bf16 rounding) are bitwise equal; biases, gammas and
    LayerNorm parameters come from column sums reduced with fp32 atomics in arrival order, whose last bits vary from
    run to run: one bf16 ulp."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = _cfg(**kw)
    x, y = _data(cfg)
    runs = []
    for mkw in (dict(grad_ckpt=True, ckpt_keep_blocks=0), dict(grad_ckpt=True, ckpt_keep_blocks=3),
                dict(grad_ckpt=False)):
        model = FSDPViT(cfg, device="cuda", dtype=torch.bfloat16, seed=4, **mkw)
        if mkw.get("ckpt_keep_blocks") == 3:
            model.keep_extras = {"P": 1, "h": 2, "g": 3}
        _randomize_gammas(model)
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


def test_init_values_one_reproduces_the_model_without_the_flag():
    """bf16(1 * W) == W: the fold is exact, so the forward (the eval logits) and every GEMM-produced weight gradient
    are bitwise those of the model without the flag.  The loss and the bias / LayerNorm gradients come out of fp32
    atomics: they may differ by what two runs of the model without the flag differ by (bounded here by one bf16 ulp
    and the loss's fp32 reordering bound)."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg1, cfg0 = _cfg(init_values=1.0), _cfg(init_values=0.0)
    x, y = _data(cfg0)
    runs = {}
    for name, cfg in (("ls", cfg1), ("plain", cfg0), ("plain2", cfg0)):
        model = FSDPViT(cfg, device="cuda", dtype=torch.bfloat16, seed=4, ckpt_keep_blocks=1)
        loss = model.forward_backward(x.cuda(), y.cuda()).item()
        grads = _named_grads(model)
        logits = model.eval()(x.cuda()).cpu()
        runs[name] = (loss, grads, logits)
    (l1, g1, z1), (l0, g0, z0), (l2, g2, _) = runs["ls"], runs["plain"], runs["plain2"]
    assert torch.equal(z1, z0)
    assert abs(l1 - l0) <= max(abs(l2 - l0), 1e-6 * abs(l0)), (l1, l0, l2)
    assert set(g1) - set(g0) == {f"blocks.{i}.ls{j}.gamma" for i in range(cfg1.num_blocks) for j in (1, 2)}
    for k in g0:
        if k.endswith(("qkv.weight", "proj.weight", "fc1.weight", "fc2.weight", "head.weight")):
            assert torch.equal(g1[k], g0[k]), k
        else:
            bound = torch.maximum((g2[k] - g0[k]).abs(), g0[k].abs() * 2.0 ** -7 + 1e-6 * g0[k].abs().max().item())
            assert ((g1[k] - g0[k]).abs() <= bound).all(), (k, (g1[k] - g0[k]).abs().max().item())


def test_cuda_graph_matches_eager():
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

    cfg = _cfg(image_size=112, embed_dim=320, num_heads=2, init_values=0.5)
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


def test_cli_trains_and_checkpoints_with_layer_scale(tmp_path):
    from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files

    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "16",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--num_epochs", "1", "--ckpt_epoch_interval", "1", "--test_epoch_interval", "100", "--init_values", "1e-5"]
    ckpt = tmp_path / "ckpt"
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(ckpt)], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "init_values=1e-05" in r.stdout
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
    full = consolidate_files(str(ckpt / "epoch_1"))
    gamma = full["blocks.1.ls2.gamma"]
    assert gamma.shape == (128,) and torch.isfinite(gamma).all()
    assert (gamma - 1e-5).abs().max().item() > 0  # two AdamW steps moved it
