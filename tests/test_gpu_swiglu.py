"""SwiGLU (--swiglu) on the GPU: the GEMM's SwiGLU forward and dSwiGLU dgrad epilogues and the memory-bound
swiglu_fwd / swiglu_bwd kernels against fp64 references computed from the same bf16 inputs, their argument checks,
the fused against the unfused route, and the model against the fp32 CPU model, across activation-keeping modes, under
CUDA graphs and through the command line.

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
BF16_HALF_ULP = 2.0 ** -8  # relative rounding error of one bf16 rounding
F32_EPS = 2.0 ** -24


def _co():
    from vit_10b_fsdp_example_b200.ops import cuda_ops

    return cuda_ops


def _silu(a):
    return a * torch.sigmoid(a)


def _dsilu(a):
    s = torch.sigmoid(a)
    return s * (1 + a * (1 - s))


def _route(monkeypatch, fused: bool):
    """Force the fused GEMM epilogues (at every K) or the plain GEMM + memory-bound kernels."""
    co = _co()
    monkeypatch.setattr(co, "SWIGLU_FWD_MIN_K", 0 if fused else 1 << 30)
    monkeypatch.setattr(co, "SWIGLU_DGRAD_K", (0, 1 << 30) if fused else (1, 0))


def _mat(rows, cols, g, scale=1.0):
    return (torch.randn(rows, cols, generator=g) * scale).bfloat16().cuda()


# ------------------------------------------------------------------------------------------------
# the GEMM epilogues against fp64
# ------------------------------------------------------------------------------------------------
# (M, K, Hd): ViT-10B-class fc1 (D 5120, Hd 4 D), DINOv2-g (D 1536, Hd = int(1536 * 5.33334) = 8192), and small /
# ragged shapes whose H' = Hd / 2 is not a multiple of 128 (or of 64) and whose M is not a multiple of 128
SHAPES = [(1024, 5120, 20480), (1000, 1536, 8192), (200, 64, 144), (129, 72, 208), (77, 256, 2064)]
CONFIGS = [(128, 1), (128, 2), (256, 1), (256, 2)]  # (block_n, cluster)


def _fp32_sum_bound(a, b):
    """Worst-case error of an fp32 dot product of length K, per output: K * 2^-24 * sum_k |a_k b_k|."""
    return a.shape[1] * F32_EPS * (a.double().abs() @ b.double().abs().t())


@pytest.mark.parametrize("block_n,cluster", CONFIGS)
@pytest.mark.parametrize("M,K,Hd", SHAPES)
def test_forward_epilogue_against_fp64(M, K, Hd, block_n, cluster):
    co = _co()
    g = torch.Generator().manual_seed(M + K + Hd)
    Hh = Hd // 2
    x, W = _mat(M, K, g), _mat(Hd, K, g, 1.0 / math.sqrt(K))
    b = (torch.randn(Hd, generator=g) * 0.5).bfloat16().cuda()
    u_ref = x.double() @ W.double().t() + b.double()
    e = _fp32_sum_bound(x, W) + 4 * F32_EPS * b.double().abs()  # accumulator + bias add, before any rounding
    a, v = u_ref[:, :Hh], u_ref[:, Hh:]
    g_ref = _silu(a) * v
    # g = bf16(silu(a') v') from the fp32 a', v': rounding + |d g / d a| e_a + |d g / d v| e_v + sigmoid approximation
    g_bound = (BF16_HALF_ULP * g_ref.abs() + _dsilu(a).abs() * v.abs() * e[:, :Hh] + _silu(a).abs() * e[:, Hh:]
               + 1e-6 * (a * v).abs() + 1e-30)
    for preact in (False, True):
        gout = torch.full((M, Hh), float("nan"), dtype=torch.bfloat16, device="cuda")
        u = torch.full((M, Hd), float("nan"), dtype=torch.bfloat16, device="cuda") if preact else None
        co.gemm_raw(x, K, 0, W, K, 0, gout, Hh, M, Hh, K, bias=b, aux_out=u, ld_aux_out=Hd, act=co.ACT_SWIGLU,
                    block_n=block_n, cluster=cluster)
        err = (gout.double() - g_ref).abs()
        assert (err <= g_bound).all(), (preact, err.max().item(), (err - g_bound).max().item())
        if preact:  # every column written, once rounded
            assert ((u.double() - u_ref).abs() <= BF16_HALF_ULP * u_ref.abs() + e).all()


@pytest.mark.parametrize("block_n,cluster", CONFIGS)
@pytest.mark.parametrize("M,K,Hd", SHAPES)
def test_dgrad_epilogue_against_fp64(M, K, Hd, block_n, cluster):
    """fc2 dgrad: dh = dt W2 [M, H'] (K = D here is the fc2 output width), du = [dh v silu'(a) | dh silu(a)]."""
    co = _co()
    g = torch.Generator().manual_seed(M * 3 + K + Hd)
    Hh = Hd // 2
    dt, W2 = _mat(M, K, g, 0.1), _mat(K, Hh, g, 1.0 / math.sqrt(K))
    u = _mat(M, Hd, g, 2.0)
    dh = dt.double() @ W2.double()
    e = _fp32_sum_bound(dt, W2.t())
    a, v = u.double()[:, :Hh], u.double()[:, Hh:]
    ref = torch.cat([dh * v * _dsilu(a), dh * _silu(a)], dim=1)
    sens = torch.cat([(v * _dsilu(a)).abs(), _silu(a).abs()], dim=1)
    bound = BF16_HALF_ULP * ref.abs() + sens * torch.cat([e, e], dim=1) + 1e-6 * dh.abs().repeat(1, 2) * (
        1 + u.double().abs() * torch.cat([v.abs(), torch.ones_like(v)], dim=1)) + 1e-30
    for want_colsum in (False, True):
        du = torch.full((M, Hd), float("nan"), dtype=torch.bfloat16, device="cuda")
        cs = torch.zeros(Hd, dtype=torch.float32, device="cuda") if want_colsum else None
        co.gemm_raw(dt, K, 0, W2, Hh, 1, du, Hd, M, Hh, K, aux_in=u, ld_aux=Hd, aux_out=du[:, Hh:], ld_aux_out=Hd,
                    act=co.ACT_DSWIGLU, colsum=cs, block_n=block_n, cluster=cluster)
        err = (du.double() - ref).abs()
        assert (err <= bound).all(), (want_colsum, err.max().item(), (err - bound).max().item())
        if want_colsum:  # sums of the stored bf16 values in fp32 (64-row partials + one atomic per 64 rows)
            want = du.double().sum(0)
            cbound = (M + 64) * F32_EPS * du.double().abs().sum(0) + 1e-30
            assert ((cs.double() - want).abs() <= cbound).all()


# ------------------------------------------------------------------------------------------------
# the memory-bound kernels against fp64, the gate swept over every finite bf16 value
# ------------------------------------------------------------------------------------------------
def _every_finite_bf16():
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    vals = bits.view(torch.bfloat16)
    return vals[torch.isfinite(vals.float())]


def test_memory_bound_kernels_on_every_bf16_gate():
    co = _co()
    gates = _every_finite_bf16()
    Hh = 256
    M = (gates.numel() + Hh - 1) // Hh
    a = torch.zeros(M * Hh, dtype=torch.bfloat16)
    a[: gates.numel()] = gates
    g = torch.Generator().manual_seed(0)
    v = (torch.rand(M, Hh, generator=g) * 2 - 1).bfloat16()
    dg = (torch.rand(M, Hh, generator=g) * 2 - 1).bfloat16()
    u = torch.cat([a.view(M, Hh), v], dim=1).cuda()
    ad, vd, dgd = a.view(M, Hh).double(), v.double(), dg.double()

    out = co.swiglu_fwd(u)
    ref = _silu(ad) * vd
    # one rounding, plus exp / rcp approximations (a few 2^-23 relative) and the flush of silu(a) < 2^-126 to zero
    bound = BF16_HALF_ULP * ref.abs() + 1e-6 * (ad * vd).abs() + 1e-30
    err = (out.cpu().double() - ref).abs()
    assert (err <= bound).all(), (err - bound).max().item()

    du = co.swiglu_bwd(dg.cuda(), u).cpu().double()
    ref = torch.cat([dgd * vd * _dsilu(ad), dgd * _silu(ad)], dim=1)
    # silu'(a) = s (1 + a (1 - s)): the fp32 1 - s carries an absolute error of ~2^-24, magnified by |a|
    bound = BF16_HALF_ULP * ref.abs() + 1e-6 * (dgd.abs() * (vd.abs() * (1 + ad.abs()) + ad.abs())).repeat(1, 2) + 1e-30
    err = (du - ref).abs()
    assert (err <= bound).all(), (err - bound).max().item()


@pytest.mark.parametrize("M,Hd", [(1, 16), (3, 48), (2048, 20480), (1000, 8192)])
def test_memory_bound_kernels_at_model_shapes(M, Hd):
    co = _co()
    g = torch.Generator().manual_seed(M + Hd)
    u = _mat(M, Hd, g, 3.0)
    dg = _mat(M, Hd // 2, g)
    a, v = u.double()[:, : Hd // 2], u.double()[:, Hd // 2:]
    ref = _silu(a) * v
    assert ((co.swiglu_fwd(u).double() - ref).abs() <= BF16_HALF_ULP * ref.abs() + 1e-6 * (a * v).abs() + 1e-30).all()
    ref = torch.cat([dg.double() * v * _dsilu(a), dg.double() * _silu(a)], dim=1)
    bound = BF16_HALF_ULP * ref.abs() + 1e-5 * dg.double().abs().repeat(1, 2) * (1 + u.double().abs()) ** 2 + 1e-30
    assert ((co.swiglu_bwd(dg, u).double() - ref).abs() <= bound).all()


# ------------------------------------------------------------------------------------------------
# the fused and unfused routes agree
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,K,Hd", [(512, 2048, 4096), (300, 64, 144)])
def test_fused_and_unfused_routes_agree(monkeypatch, M, K, Hd):
    """The fused route computes g from the fp32 pre-activation, the unfused one from its bf16 rounding."""
    co = _co()
    g = torch.Generator().manual_seed(5)
    x, W = _mat(M, K, g), _mat(Hd, K, g, 1.0 / math.sqrt(K))
    b = (torch.randn(Hd, generator=g) * 0.5).bfloat16().cuda()
    dt, W2 = _mat(M, 96, g, 0.1), _mat(96, Hd // 2, g, 0.1)
    res = {}
    for route in ("fused", "unfused"):
        _route(monkeypatch, route == "fused")
        gg, u = co.linear_fwd(x, W, b, act="swiglu", want_preact=True)
        du, cs = co.linear_dgrad(dt, W2, dswiglu_preact=u, want_colsum=True)
        res[route] = (gg.double(), u.double(), du.double(), cs.double())
    (g0, u0, d0, c0), (g1, u1, d1, c1) = res["fused"], res["unfused"]
    # both store bf16(the same fp32 accumulator + bias): one rounding each, possibly of differently ordered sums
    assert ((u0 - u1).abs() <= BF16_HALF_ULP * (u0.abs() + u1.abs()) + 1e-6).all()
    a, v = u0[:, : Hd // 2], u0[:, Hd // 2:]
    # g: each route rounds once, and the unfused one reads a and v rounded to bf16 (|a|, |v| * 2^-8 each)
    gb = BF16_HALF_ULP * (g0.abs() + g1.abs() + (_dsilu(a) * v * a).abs() + (_silu(a) * v).abs()) + 1e-6
    assert ((g0 - g1).abs() <= gb).all(), ((g0 - g1).abs() - gb).max().item()
    # du: each route rounds once, the unfused one also rounds dh (a relative 2^-8 of every term)
    db = 2 * BF16_HALF_ULP * (d0.abs() + d1.abs()) + 1e-6
    assert ((d0 - d1).abs() <= db).all(), ((d0 - d1).abs() - db).max().item()
    assert ((c0 - c1).abs() <= 2 * BF16_HALF_ULP * (d0.abs().sum(0) + d1.abs().sum(0)) + 1e-4).all()


def test_rejects_bad_arguments():
    co = _co()
    g = torch.Generator().manual_seed(1)
    M, K, Hd = 128, 64, 256
    Hh = Hd // 2
    x, W, b = _mat(M, K, g), _mat(Hd, K, g), _mat(1, Hd, g)[0]
    out = torch.empty(M, Hh, dtype=torch.bfloat16, device="cuda")
    fwd = dict(act=co.ACT_SWIGLU)
    cases = [
        (dict(residual=out, ld_res=Hh), "SwiGLU epilogues take no residual"),
        (dict(row_scale=torch.ones(M, device="cuda"), rows_per_scale=1), "SwiGLU epilogues take no row_scale"),
        (dict(batch=(2, 1, 0, 0, 0, 0, M * Hh, 0)), "SwiGLU epilogues take no batched operands"),
        (dict(ag=[2, 0, Hd // 2, Hd // 2 * K * 2, out.data_ptr(), out.data_ptr(), W.data_ptr(), W.data_ptr()]),
         "SwiGLU epilogues take no AG fusion"),
        (dict(colsum=torch.zeros(Hd, device="cuda")), "SwiGLU forward takes no aux_in and no column sums"),
        (dict(block_n=64), "SwiGLU block_n must be 128 or 256"),
    ]
    for kw, msg in cases:
        with pytest.raises(RuntimeError, match=msg):
            co.gemm_raw(x, K, 0, W, K, 0, out, Hh, M, Hh, K, bias=b, **dict(fwd, **kw))
    with pytest.raises(RuntimeError, match="SwiGLU forward needs K-major A and B"):
        co.gemm_raw(x, K, 0, W, K, 1, out, Hh, M, Hh, K, act=co.ACT_SWIGLU)
    with pytest.raises(RuntimeError, match=r"multiple of 8 \(Hd % 16 == 0\)"):
        co.gemm_raw(x, K, 0, W, K, 0, out, Hh, M, 60, K, act=co.ACT_SWIGLU)
    du = torch.empty(M, Hd, dtype=torch.bfloat16, device="cuda")
    dt, W2 = _mat(M, K, g), _mat(K, Hh, g)
    with pytest.raises(RuntimeError, match="dSwiGLU needs aux_in"):
        co.gemm_raw(dt, K, 0, W2, Hh, 1, du, Hd, M, Hh, K, act=co.ACT_DSWIGLU, aux_out=du[:, Hh:], ld_aux_out=Hd)
    with pytest.raises(RuntimeError, match="dSwiGLU needs K-major A and MN-major B"):
        co.gemm_raw(dt, K, 0, W2, Hh, 0, du, Hd, M, Hh, K, act=co.ACT_DSWIGLU, aux_in=du, ld_aux=Hd,
                    aux_out=du[:, Hh:], ld_aux_out=Hd)
    with pytest.raises(RuntimeError, match="Hd must be a multiple of 16"):
        co._C.swiglu_fwd(torch.zeros(4, 24, dtype=torch.bfloat16, device="cuda"),
                         torch.zeros(4, 12, dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(RuntimeError, match=r"g must be \[M, Hd / 2\]"):
        co._C.swiglu_fwd(torch.zeros(4, 32, dtype=torch.bfloat16, device="cuda"),
                         torch.zeros(4, 32, dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(RuntimeError, match=r"du \[M, Hd\]"):
        co._C.swiglu_bwd(torch.zeros(4, 16, dtype=torch.bfloat16, device="cuda"),
                         torch.zeros(4, 32, dtype=torch.bfloat16, device="cuda"),
                         torch.zeros(4, 16, dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(ValueError, match="fc1 width Hd must be a multiple of 16"):
        co.linear_fwd(x, W[:200], act="swiglu")


# ------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------
def _cfg(**kw):
    from vit_10b_fsdp_example_b200.config import ViTConfig

    d = dict(image_size=224, patch_size=14, embed_dim=256, num_heads=4, num_blocks=3, mlp_ratio=4.0, num_classes=96,
             swiglu=True)
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


# fused: N = 256, hd 64 (wgmma attention) and the SwiGLU GEMM epilogues;
# unfused: N = 225, hd 80 (GEMM + softmax) and the plain GEMM + swiglu_fwd / swiglu_bwd
ROUTES = {"fused": (dict(), True), "unfused": (dict(image_size=210, embed_dim=320), False)}


@pytest.mark.parametrize("route", list(ROUTES))
def test_model_matches_the_fp32_cpu_model(monkeypatch, route):
    from vit_10b_fsdp_example_b200.ops import cuda_ops
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    kw, fused = ROUTES[route]
    _route(monkeypatch, fused)
    cfg = _cfg(**kw)
    assert cuda_ops.use_flash(cfg.num_patches, cfg.head_dim) == (route == "fused")
    x, y = _data(cfg)
    for keep in (0, 3):
        res = []
        for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
            model = FSDPViT(cfg, device=dev, dtype=dtype, seed=4, ckpt_keep_blocks=keep)
            loss = model.forward_backward(x.to(dev), y.to(dev)).item()
            res.append((loss, _named_grads(model)))
        (loss_ref, g_ref), (loss, grads) = res
        assert math.isfinite(loss) and abs(loss - loss_ref) < 1e-2 * abs(loss_ref) + 1e-2, (keep, loss, loss_ref)
        assert g_ref["blocks.0.mlp.fc2.weight"].shape == (cfg.embed_dim, cfg.hidden_dim // 2)
        for k in g_ref:
            a, b = g_ref[k], grads[k]
            # bf16 activations and weights through three blocks: 5 % of the gradient's norm, as for the other flags
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (keep, k)


@pytest.mark.parametrize("kw,fused", [(dict(), True), (dict(), False), (dict(mlp_dropout=0.1, att_dropout=0.1), True),
                                      (dict(drop_path_rate=0.5, init_values=1e-5, qk_norm=True), True)])
def test_checkpointed_kept_and_uncheckpointed_blocks_give_the_same_gradients(monkeypatch, kw, fused):
    """GEMM-produced weight gradients are bitwise equal; biases and LayerNorm parameters come from column sums reduced
    with fp32 atomics in arrival order, whose last bits vary from run to run: one bf16 ulp."""
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    _route(monkeypatch, fused)
    cfg = _cfg(**kw)
    x, y = _data(cfg)
    runs = []
    for mkw in (dict(grad_ckpt=True, ckpt_keep_blocks=0), dict(grad_ckpt=True, ckpt_keep_blocks=3),
                dict(grad_ckpt=False)):
        model = FSDPViT(cfg, device="cuda", dtype=torch.bfloat16, seed=4, **mkw)
        if mkw.get("ckpt_keep_blocks") == 3:
            model.keep_extras = {"P": 1, "h": 2, "g": 3}
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


def test_cuda_graph_matches_eager(monkeypatch):
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

    _route(monkeypatch, True)
    cfg = _cfg(image_size=112, embed_dim=320, num_heads=2, init_values=0.5, class_token=True, reg_tokens=4)
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


def test_cli_trains_checkpoints_consolidates_and_evaluates(tmp_path):
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "16",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--num_epochs", "1", "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--swiglu",
            "--class_token", "--reg_tokens", "4", "--init_values", "1e-5"]
    ckpt = tmp_path / "ckpt"
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(ckpt)], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
    assert re.search(r"accuracy", r.stdout, re.IGNORECASE), r.stdout[-2000:]
    full = consolidate_files(str(ckpt / "epoch_1"))
    assert full["blocks.1.mlp.fc1.weight"].shape == (512, 128) and full["blocks.1.mlp.fc2.weight"].shape == (128, 256)
    cfg = ViTConfig(image_size=224, patch_size=16, embed_dim=128, num_heads=2, num_blocks=2, num_classes=10,
                    swiglu=True, class_token=True, reg_tokens=4, init_values=1e-5)
    plain = PlainViT(cfg).eval()
    plain.load_state_dict(full, strict=True)
    with torch.no_grad():
        assert torch.isfinite(plain(torch.randn(2, 3, 224, 224))).all()
