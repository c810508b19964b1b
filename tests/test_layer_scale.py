"""LayerScale (--init_values): timm LayerScale semantics, the torch_ops reference of the fold and of its weight-side
backward, the engine against an fp64 autograd oracle, FSDP equivalence, checkpoints, CLI and the build of the sm_90a
kernels.

The oracle writes the specification literally: x1 = x + gamma1 * branch1, y = x1 + gamma2 * branch2.  The engine
instead folds gamma into the proj / fc2 weight and recovers dgamma from the weight gradient, so every engine check here
randomises the gammas (mixed signs, magnitude about 1): at the 1e-5 of a real run the branches barely move the loss and
a wrong dgamma or dW would go unnoticed."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from dist_worker import launch
from helpers import full_grads_of, full_params_of, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT

IMAGES = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(7))
TARGET = torch.tensor([1, 5, 7, 2])


def ls_cfg(**kw):
    return tiny_cfg(**dict(dict(init_values=1e-5), **kw))


def random_gamma(shape, g):
    """U(0.5, 1.5) with random signs."""
    sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
    return sign * (0.5 + torch.rand(shape, generator=g))


def randomize_gammas(model, seed=0):
    g = torch.Generator().manual_seed(seed)
    full = full_params_of(model)
    for k, v in full.items():
        if k.endswith(("ls1.gamma", "ls2.gamma")):
            full[k] = random_gamma(v.shape, g)
        elif ".q_norm." in k or ".k_norm." in k:
            full[k] = (1.0 if k.endswith("weight") else 0.0) + 0.5 * torch.randn(v.shape, generator=g)
    model.load_full_state_dict(full)


# ------------------------------------------------------------------------------------------------
# the ops against fp64
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,K,D", [(7, 8, 5), (33, 13, 9), (5, 1, 3), (64, 40, 16), (17, 1027, 4), (3, 24, 1)])
def test_ops_against_fp64(R, K, D):
    """u = a W^T + b [R, D]; the reference computes dgamma directly as sum_r dy'[r, c] u[r, c], so the identity
    dgamma_c = sum_k W[c, k] M[c, k] + b_c S_c that the op uses is itself under test."""
    g = torch.Generator().manual_seed(R * 1000 + K * 10 + D)
    a = torch.randn(R, K, generator=g)
    W = torch.randn(D, K, generator=g)
    b = torch.randn(D, generator=g)
    gamma = random_gamma(D, g)
    gamma[0] = 1e-5
    dy = torch.randn(R, D, generator=g)

    Wg, bg = torch_ops.layer_scale_fold(W, b, gamma)
    ref = a.double() @ (gamma.double()[:, None] * W.double()).t() + gamma.double() * b.double()
    got = a.double() @ Wg.double().t() + bg.double()
    assert (got - ref).abs().max() <= 1e-5 * (ref.abs().max() + 1)
    assert torch.allclose(Wg.double(), gamma.double()[:, None] * W.double(), rtol=1e-6, atol=0)

    # backward: M = dy^T a is what the wgrad writes, S = colsum(dy) what the code already has
    u = a.double() @ W.double().t() + b.double()
    M = dy.t() @ a
    S = dy.sum(0)
    dW = M.clone()
    Wg2, db, dgamma = torch_ops.layer_scale_bwd(W, b, gamma, dW, S)
    assert torch.equal(Wg2, Wg)
    want_dgamma = (dy.double() * u).sum(0)
    scale = (dy.double().abs() * u.abs()).sum(0)
    assert ((dgamma.double() - want_dgamma).abs() <= 1e-5 * scale + 1e-6).all(), (dgamma, want_dgamma)
    want_dW = gamma.double()[:, None] * (dy.double().t() @ a.double())
    assert (dW.double() - want_dW).abs().max() <= 1e-5 * (want_dW.abs().max() + 1)
    assert torch.allclose(db.double(), gamma.double() * dy.double().sum(0), rtol=1e-5, atol=1e-6)

    # and all of it against autograd on the specification gamma * (a W^T + b)
    pa, pw, pb, pg = (t.double().requires_grad_(True) for t in (a, W, b, gamma))
    (pg * F.linear(pa, pw, pb)).backward(dy.double())
    assert (dW.double() - pw.grad).abs().max() <= 1e-5 * (pw.grad.abs().max() + 1)
    assert torch.allclose(db.double(), pb.grad, rtol=1e-5, atol=1e-6)
    assert ((dgamma.double() - pg.grad).abs() <= 1e-5 * scale + 1e-6).all()
    assert (dy.double() @ Wg.double() - pa.grad).abs().max() <= 1e-5 * (pa.grad.abs().max() + 1)


def test_ops_round_once_in_bf16():
    g = torch.Generator().manual_seed(0)
    W, b = torch.randn(6, 19, generator=g).bfloat16(), torch.randn(6, generator=g).bfloat16()
    gamma = random_gamma(6, g).bfloat16()
    Wg, bg = torch_ops.layer_scale_fold(W, b, gamma)
    assert Wg.dtype == bg.dtype == torch.bfloat16
    assert torch.equal(Wg, (W.float() * gamma.float()[:, None]).bfloat16())
    ones = torch.ones(6, dtype=torch.bfloat16)
    assert torch.equal(torch_ops.layer_scale_fold(W, b, ones)[0], W)  # gamma = 1 is exact
    dW = torch.randn(6, 19, generator=g).bfloat16()
    M = dW.clone()
    _, db, dgamma = torch_ops.layer_scale_bwd(W, b, gamma, dW, torch.ones(6))
    assert dW.dtype == torch.bfloat16 and db.dtype == dgamma.dtype == torch.float32
    assert torch.equal(dW, (M.float() * gamma.float()[:, None]).bfloat16())


# ------------------------------------------------------------------------------------------------
# the engine against the fp64 oracle
# ------------------------------------------------------------------------------------------------
def autograd_vit_loss_ls(cfg, params, images, target, masks=None):
    """timm ViT with LayerScale (and QK normalisation when cfg.qk_norm).  masks: optional per-block dict of
    multiplicative dropout / drop-path factors {"att": [B,H,N,N], "proj", "fc1", "fc2": like their tensors,
    "sa", "sm": [B,1,1]}."""
    B = images.shape[0]
    N, D, H, hd, P = cfg.num_patches, cfg.embed_dim, cfg.num_heads, cfg.head_dim, cfg.patch_size
    w = params["patch_embed.proj.weight"][:, : cfg.patch_k].reshape(D, 3, P, P)
    x = F.conv2d(images, w, params["patch_embed.proj.bias"], stride=P).flatten(2).transpose(1, 2)
    x = x + params["pos_embed"].view(1, N, D)
    for i in range(cfg.num_blocks):
        g = lambda n: params[f"blocks.{i}.{n}"]  # noqa: E731
        mk = (masks or [None] * cfg.num_blocks)[i] or {}
        m = lambda name, t: t * mk[name] if name in mk else t  # noqa: E731
        h = F.layer_norm(x, (D,), g("norm1.weight"), g("norm1.bias"), 1e-5)
        q, k, v = F.linear(h, g("attn.qkv.weight"), g("attn.qkv.bias")).reshape(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
        if cfg.qk_norm:
            q = F.layer_norm(q, (hd,), g("attn.q_norm.weight"), g("attn.q_norm.bias"), 1e-5)
            k = F.layer_norm(k, (hd,), g("attn.k_norm.weight"), g("attn.k_norm.bias"), 1e-5)
        att = m("att", ((q @ k.transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1))
        a = (att @ v).transpose(1, 2).reshape(B, N, D)
        x = x + g("ls1.gamma") * m("sa", m("proj", F.linear(a, g("attn.proj.weight"), g("attn.proj.bias"))))
        h = F.layer_norm(x, (D,), g("norm2.weight"), g("norm2.bias"), 1e-5)
        h = m("fc1", F.gelu(F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias"))))
        x = x + g("ls2.gamma") * m("sm", m("fc2", F.linear(h, g("mlp.fc2.weight"), g("mlp.fc2.bias"))))
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x.mean(dim=1), params["head.weight"], params["head.bias"])
    return F.cross_entropy(logits, target), logits


def _check_against_oracle(model, images, target, masks=None):
    loss = model.forward_backward(images, target)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    assert params["blocks.0.ls1.gamma"].abs().min() >= 0.5  # randomised, not the 1e-5 start
    ref_loss, ref_logits = autograd_vit_loss_ls(model.cfg, params, images.double(), target, masks)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 1e-5, (loss.item(), ref_loss.item())
    for name, p in params.items():
        g = p.grad if p.grad is not None else torch.zeros_like(p)
        err = (got[name].double() - g).abs().max().item()
        if name.endswith("k_norm.bias"):  # exactly zero: the softmax cancels q . b_k; fp32 rounding is left
            assert g.abs().max().item() < 1e-12 and err < 1e-7, f"{name}: err {err}"
            continue
        scale = g.abs().max().item() + 1e-8
        assert err / scale < 2e-4, f"{name}: err {err} scale {scale}"
    return ref_logits


@pytest.mark.parametrize("grad_ckpt,keep,flatten", [(True, 0, False), (False, 0, False), (True, 0, True),
                                                    (False, 0, True), (True, 1, False), (True, 99, False)])
def test_engine_matches_autograd(grad_ckpt, keep, flatten):
    cfg = ls_cfg()
    model = FSDPViT(cfg, dtype=torch.float32, grad_ckpt=grad_ckpt, ckpt_keep_blocks=keep, flatten_parameters=flatten,
                    seed=3)
    randomize_gammas(model)
    images = torch.randn(4, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(1))
    ref_logits = _check_against_oracle(model, images, TARGET)
    assert torch.allclose(model.eval()(images).double(), ref_logits.detach(), atol=1e-4)


@pytest.mark.parametrize("extras", [{"P": 99, "h": 99, "g": 99}, {"P": 1, "h": 0, "g": 1}, {"P": 0, "h": 99, "g": 0}])
def test_kept_blocks_with_extras_match_autograd(extras):
    model = FSDPViT(ls_cfg(), dtype=torch.float32, grad_ckpt=True, ckpt_keep_blocks=99, seed=3)
    model.keep_extras = extras
    randomize_gammas(model, seed=1)
    _check_against_oracle(model, IMAGES, TARGET)


@pytest.mark.parametrize("qk_norm", [False, True])
def test_flash_style_path_and_qk_norm_match_autograd(monkeypatch, qk_norm):
    monkeypatch.setattr(torch_ops, "FLASH_ATTENTION", True)
    for kw in (dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)):
        model = FSDPViT(ls_cfg(qk_norm=qk_norm), dtype=torch.float32, seed=3, **kw)
        randomize_gammas(model, seed=2)
        _check_against_oracle(model, IMAGES, TARGET)


def _model_masks(model, B):
    """The multiplicative dropout / drop-path factors the model's blocks draw in its next training step."""
    cfg, ctx = model.cfg, model.drop
    N, H, D = cfg.num_patches, cfg.num_heads, cfg.embed_dim
    pa, pm = cfg.att_dropout, cfg.mlp_dropout
    out = []
    for i, rate in enumerate(vit.drop_path_rates(cfg)):
        site = i * 8
        m = {}
        if pa > 0:
            m["att"] = torch_ops.dropout(torch.ones(B * H, N, N, dtype=torch.float64), pa, ctx.key(site)).view(B, H, N, N)
        if pm > 0:
            m["proj"] = torch_ops.dropout(torch.ones(B * N, D, dtype=torch.float64), pm, ctx.key(site + 1)).view(B, N, D)
            m["fc1"] = torch_ops.dropout(torch.ones(B * N, cfg.hidden_dim, dtype=torch.float64), pm,
                                         ctx.key(site + 2)).view(B, N, -1)
            m["fc2"] = torch_ops.dropout(torch.ones(B * N, D, dtype=torch.float64), pm, ctx.key(site + 3)).view(B, N, D)
        if rate > 0:
            m["sa"] = torch_ops.drop_path_scale(ctx.key(site + 4), rate, B, model.rank * B, "cpu").double().view(B, 1, 1)
            m["sm"] = torch_ops.drop_path_scale(ctx.key(site + 5), rate, B, model.rank * B, "cpu").double().view(B, 1, 1)
        out.append(m)
    return out


@pytest.mark.parametrize("kw", [dict(att_dropout=0.2), dict(mlp_dropout=0.2), dict(drop_path_rate=0.5),
                                dict(att_dropout=0.1, mlp_dropout=0.1, drop_path_rate=0.5)])
@pytest.mark.parametrize("mode", [dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)])
def test_composes_with_dropout_and_drop_path(kw, mode):
    cfg = ls_cfg(num_blocks=4, **kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3, **mode)
    randomize_gammas(model, seed=3)
    images = torch.randn(8, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(2))
    target = torch.randint(0, 10, (8,), generator=torch.Generator().manual_seed(2))
    _check_against_oracle(model, images, target, _model_masks(model, 8))


# ------------------------------------------------------------------------------------------------
# default behaviour, parameters, config
# ------------------------------------------------------------------------------------------------
def test_flag_off_calls_nothing_new(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("layer_scale op called without --init_values")

    monkeypatch.setattr(torch_ops, "layer_scale_fold", boom)
    monkeypatch.setattr(torch_ops, "layer_scale_bwd", boom)
    for kw in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
        model = FSDPViT(tiny_cfg(drop_path_rate=0.3, mlp_dropout=0.1), dtype=torch.float32, seed=3, **kw)
        model.forward_backward(IMAGES, TARGET)
        model.eval()(IMAGES)
    assert not any(n.startswith("ls") for n, _ in vit.block_param_specs(tiny_cfg()))


def test_parameters_order_init_and_count():
    cfg = ls_cfg(init_values=1e-4)
    names = [n for n, _ in vit.block_param_specs(cfg)]
    assert names[names.index("attn.proj.bias") + 1] == "ls1.gamma"
    assert names[names.index("mlp.fc2.bias") + 1] == "ls2.gamma" and names[-1] == "ls2.gamma"
    assert all(s == (cfg.embed_dim,) for n, s in vit.block_param_specs(cfg) if n.startswith("ls"))
    assert set(vit.init_block_params(cfg, torch.Generator().manual_seed(0))) == set(names)
    a = full_params_of(FSDPViT(cfg, dtype=torch.float32, seed=5))
    b = full_params_of(FSDPViT(tiny_cfg(), dtype=torch.float32, seed=5))
    for k, v in a.items():
        if k.endswith(("ls1.gamma", "ls2.gamma")):
            assert torch.equal(v, torch.full_like(v, 1e-4)), k
        else:
            assert torch.equal(v, b[k]), k  # the gammas draw nothing: every other parameter is the same-seed one
    assert set(a) - set(b) == {f"blocks.{i}.ls{j}.gamma" for i in range(cfg.num_blocks) for j in (1, 2)}
    assert cfg.block_numel() == tiny_cfg().block_numel() + 2 * cfg.embed_dim
    assert cfg.block_numel() == sum(torch.Size(s).numel() for _, s in vit.block_param_specs(cfg))
    assert ViTConfig(init_values=1e-5).block_numel() - ViTConfig().block_numel() == 2 * 5120
    assert ViTConfig(init_values=1e-5).flops_per_image() == ViTConfig().flops_per_image()
    qk = ls_cfg(qk_norm=True)
    assert qk.block_numel() == sum(torch.Size(s).numel() for _, s in vit.block_param_specs(qk))


def test_lean_bytes_unchanged():
    a = FSDPViT(ls_cfg(), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    assert a.lean_bytes_per_block(4) == b.lean_bytes_per_block(4)


def test_init_values_one_reproduces_the_model_without_the_flag():
    a = FSDPViT(ls_cfg(init_values=1.0), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    assert abs(a.forward_backward(IMAGES, TARGET).item() - b.forward_backward(IMAGES, TARGET).item()) < 1e-6
    ga, gb = full_grads_of(a), full_grads_of(b)
    for k, v in gb.items():
        assert torch.allclose(ga[k], v, rtol=1e-5, atol=1e-7), k


def test_cli_parsing_and_rejections():
    assert parse_args([]).init_values == 0.0
    assert ViTConfig.from_args(parse_args([])).init_values == 0.0
    args = parse_args(["--init_values", "1e-5"])
    assert args.init_values == 1e-5 and ViTConfig.from_args(args).init_values == 1e-5
    for bad in ("-1e-5", "nan", "inf"):
        with pytest.raises(SystemExit):
            parse_args(["--init_values", bad])
    for bad in (-1e-5, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="init_values must be a finite number >= 0"):
            tiny_cfg(init_values=bad)


# ------------------------------------------------------------------------------------------------
# FSDP equivalence and checkpoints
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ls_baseline(tmp_path_factory):
    out = tmp_path_factory.mktemp("ls_base") / "r.json"
    return launch(1, {"model": {"init_values": 0.5}, "steps": 4}, str(out))


def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.mark.parametrize("opts", [{}, {"flatten": True}])
def test_two_ranks_reproduce_one(opts, ls_baseline, tmp_path):
    res = launch(2, dict(opts, model={"init_values": 0.5}, steps=4), str(tmp_path / "r.json"))
    _close(res["losses"], ls_baseline["losses"])
    _close(res["norms"], ls_baseline["norms"], tol=1e-4)


def test_resume_equals_uninterrupted(tmp_path):
    d = str(tmp_path)
    model = {"init_values": 0.5}
    full = launch(2, {"model": model, "steps": 5}, os.path.join(d, "full.json"))
    launch(2, {"model": model, "steps": 3, "save_at": 3, "save_path": os.path.join(d, "e1_rank_{rank}.ckpt")},
           os.path.join(d, "part.json"))
    rest = launch(2, {"model": model, "steps": 5, "resume_from": os.path.join(d, "e1_rank_{rank}.ckpt"),
                      "resume_step": 3}, os.path.join(d, "rest.json"))
    for a, b in zip(rest["losses"], full["losses"][3:]):
        assert abs(a - b) < 1e-6


def test_consolidated_checkpoint_loads_into_plain_vit_and_back(tmp_path):
    from vit_10b_fsdp_example_b200.models.plain import PlainViT

    d = str(tmp_path)
    prefix = os.path.join(d, "epoch_1")
    # two training steps so that the gammas are no longer their initial value
    launch(2, {"model": {"init_values": 0.5}, "steps": 2, "seed": 7, "dump_state": prefix + "_rank_{rank}.ckpt"},
           os.path.join(d, "r.json"))
    full = consolidate_files(prefix, save_path=prefix + "_full.pth")
    cfg = ls_cfg(init_values=0.5)
    assert full["blocks.0.ls1.gamma"].shape == (cfg.embed_dim,)
    assert not torch.equal(full["blocks.0.ls2.gamma"], torch.full((cfg.embed_dim,), 0.5))
    engine = FSDPViT(cfg, dtype=torch.float32, seed=99)
    engine.load_full_state_dict(full)
    plain = PlainViT.from_consolidated(prefix + "_full.pth", cfg).eval()
    assert set(plain.state_dict()) == set(full)
    block0 = [k for k in full if k.startswith("blocks.0.")]
    assert block0 == [f"blocks.0.{k}" for k in plain.blocks[0].state_dict()]  # timm's Block order
    images = torch.randn(3, 3, cfg.image_size, cfg.image_size)
    with torch.no_grad():
        want = plain(images)
    got = engine.eval()(images)
    assert torch.allclose(got, want, atol=1e-4), (got - want).abs().max()
    # and back: the plain model's state_dict loads into the engine (any init_values > 0: the gammas are loaded)
    back = FSDPViT(ls_cfg(init_values=1e-5), dtype=torch.float32, seed=5)
    back.load_full_state_dict(plain.state_dict())
    assert torch.allclose(back.eval()(images), want, atol=1e-4)


def test_full_checkpoint_refusals():
    with_ls = full_params_of(FSDPViT(ls_cfg(), dtype=torch.float32, seed=1))
    without = full_params_of(FSDPViT(tiny_cfg(), dtype=torch.float32, seed=1))
    with pytest.raises(ValueError, match=r"uses --init_values \(LayerScale\), but the checkpoint has no ls1.gamma"):
        FSDPViT(ls_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(without)
    with pytest.raises(ValueError, match="trained with LayerScale\\): pass --init_values to load it"):
        FSDPViT(tiny_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(with_ls)
    FSDPViT(ls_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(with_ls)  # the matching pairs load
    FSDPViT(tiny_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(without)


@pytest.mark.parametrize("direction", ["flag_without_gammas", "gammas_without_flag"])
def test_full_checkpoint_refusal_through_the_cli(tmp_path, direction):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    small = dict(num_blocks=2, embed_dim=32, num_heads=2)
    saved_cfg = tiny_cfg(**small) if direction == "flag_without_gammas" else ls_cfg(**small)
    sd = full_params_of(FSDPViT(saved_cfg, dtype=torch.float32, seed=1))
    sd["pos_embed"] = sd["pos_embed"][None]  # the consolidated (timm) shape [1, N, D]
    full = str(tmp_path / "plain.pth")
    torch.save({"model": sd}, full)
    args = ["run_vit_training.py", "--fake_data", "--device", "cpu", "--nproc", "1", "--image_size", "32",
            "--patch_size", "8", "--embed_dim", "32", "--num_heads", "2", "--num_blocks", "2", "--mlp_ratio", "2",
            "--num_classes", "10", "--batch_size", "4", "--max_steps", "1", "--num_workers", "0", "--num_epochs", "1",
            "--ckpt_dir", str(tmp_path / "c"), "--init_from_full_ckpt", full]
    if direction == "flag_without_gammas":
        args += ["--init_values", "1e-5"]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, *args], cwd=root, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0
    want = ("uses --init_values (LayerScale), but the checkpoint has no ls1.gamma"
            if direction == "flag_without_gammas" else "pass --init_values to load it")
    assert want in r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------
# build: the new kernels compile for sm_90a without spills or calls
# ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")),
                    reason="needs nvcc")
def test_layer_scale_kernels_compile_for_sm90a_without_spills(tmp_path):
    import shutil

    from vit_10b_fsdp_example_b200 import build_ext

    nvcc = os.path.join(build_ext._cuda_home(), "bin", "nvcc")
    res = subprocess.run([nvcc, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, "layer_scale.cu"), "-o", str(tmp_path / "l.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = (res.stdout + res.stderr).splitlines()
    found = {}
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln:
            assert "sm_90a" in ln
            found[ln.split("'")[1]] = next(x for x in lines[i + 1:] if "spill stores" in x)
    assert len(found) == 2 and all("layer_scale_kernel" in k for k in found), found
    assert all("0 bytes spill stores, 0 bytes spill loads" in v for v in found.values()), found
    if shutil.which("cuobjdump"):
        sass = subprocess.run(["cuobjdump", "-sass", str(tmp_path / "l.o")], capture_output=True, text=True).stdout
        assert "layer_scale_kernel" in sass and " CALL" not in sass
