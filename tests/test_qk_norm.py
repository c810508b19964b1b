"""QK normalisation (--qk_norm): timm Attention(qk_norm=True) semantics, the torch_ops reference, the hand-written
backward against autograd, FSDP equivalence, checkpoints, CLI and the build of the sm_90a kernels.

The oracle below implements the specification literally: split qkv into [B, H, N, hd] q, k, v, F.layer_norm over the
last dim of q and k (one weight and bias of size hd per block), then softmax(q k^T * hd^-0.5) v."""
import os
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

from dist_worker import launch
from helpers import full_grads_of, full_params_of, tiny_cfg
from vit_10b_fsdp_example_b200.config import ViTConfig, parse_args
from vit_10b_fsdp_example_b200.consolidate_sharded_ckpts import consolidate_files
from vit_10b_fsdp_example_b200.models import vit
from vit_10b_fsdp_example_b200.ops import torch_ops
from vit_10b_fsdp_example_b200.parallel import FSDPViT, GraphedTrainStep, ShardedAdamW

IMAGES = torch.randn(4, 3, 32, 32, generator=torch.Generator().manual_seed(7))
TARGET = torch.tensor([1, 5, 7, 2])


def qk_cfg(**kw):
    return tiny_cfg(qk_norm=True, **kw)


def randomize_qk_params(model, seed=0):
    """The norms start as ones / zeros, which hides a transposed or mis-indexed weight: give them random values."""
    g = torch.Generator().manual_seed(seed)
    full = full_params_of(model)
    for k, v in full.items():
        if ".q_norm." in k or ".k_norm." in k:
            full[k] = (1.0 if k.endswith("weight") else 0.0) + 0.5 * torch.randn(v.shape, generator=g)
    model.load_full_state_dict(full)


# ------------------------------------------------------------------------------------------------
# fp64 autograd oracle of the whole model
# ------------------------------------------------------------------------------------------------
def autograd_vit_loss_qk(cfg, params, images, target, masks=None):
    """timm ViT whose attention is Attention(qk_norm=True).  masks: optional per-block dict of multiplicative dropout /
    drop-path factors {"att": [B,H,N,N], "proj", "fc1", "fc2": like their tensors, "sa", "sm": [B,1,1]}."""
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
        qkv = F.linear(h, g("attn.qkv.weight"), g("attn.qkv.bias")).reshape(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
        q = F.layer_norm(qkv[0], (hd,), g("attn.q_norm.weight"), g("attn.q_norm.bias"), 1e-5)
        k = F.layer_norm(qkv[1], (hd,), g("attn.k_norm.weight"), g("attn.k_norm.bias"), 1e-5)
        att = m("att", ((q @ k.transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1))
        a = (att @ qkv[2]).transpose(1, 2).reshape(B, N, D)
        x = x + m("sa", m("proj", F.linear(a, g("attn.proj.weight"), g("attn.proj.bias"))))
        h = F.layer_norm(x, (D,), g("norm2.weight"), g("norm2.bias"), 1e-5)
        h = m("fc1", F.gelu(F.linear(h, g("mlp.fc1.weight"), g("mlp.fc1.bias"))))
        x = x + m("sm", m("fc2", F.linear(h, g("mlp.fc2.weight"), g("mlp.fc2.bias"))))
    x = F.layer_norm(x, (D,), params["norm.weight"], params["norm.bias"], 1e-6)
    logits = F.linear(x.mean(dim=1), params["head.weight"], params["head.bias"])
    return F.cross_entropy(logits, target), logits


def _check_against_oracle(model, images, target, masks=None):
    loss = model.forward_backward(images, target)
    got = full_grads_of(model)
    params = {k: v.double().requires_grad_(True) for k, v in full_params_of(model).items()}
    ref_loss, ref_logits = autograd_vit_loss_qk(model.cfg, params, images.double(), target, masks)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) < 1e-5, (loss.item(), ref_loss.item())
    assert any(".q_norm." in k for k in params)
    for name, p in params.items():
        g = p.grad if p.grad is not None else torch.zeros_like(p)
        err = (got[name].double() - g).abs().max().item()
        if name.endswith("k_norm.bias"):
            # exactly zero: the k bias adds q . b_k to every score of a row, which the softmax cancels; what is left
            # is fp32 rounding
            assert g.abs().max().item() < 1e-12 and err < 1e-7, f"{name}: err {err}"
            continue
        scale = g.abs().max().item() + 1e-8
        assert err / scale < 2e-4, f"{name}: err {err} scale {scale}"
    return ref_logits


# ------------------------------------------------------------------------------------------------
# the ops against autograd on F.layer_norm, in fp64
# ------------------------------------------------------------------------------------------------
def _rel(got, want):
    return (got.double() - want).abs().max().item() / (want.abs().max().item() + 1e-30)


@pytest.mark.parametrize("T,H,hd", [(5, 1, 8), (7, 3, 16), (12, 4, 40), (3, 2, 160), (1, 5, 64), (9, 2, 256)])
def test_ops_match_autograd_layer_norm(T, H, hd):
    """The fp32 reference ops against fp64 autograd through F.layer_norm over the last dim of [T, H, hd] q and k."""
    g = torch.Generator().manual_seed(T * 100 + H * 10 + hd)
    D = H * hd
    qkv = torch.randn(T, 3 * D, generator=g) * 3 + 1
    qkv[0, :hd] = 2.5  # a constant q row
    qkv[-1, D + (H - 1) * hd: D + H * hd] = -1.0  # a constant k row
    qkv[1 % T, hd // 2: hd] += 100.0  # |mean| >> std on part of a row
    wq, bq, wk, bk = (torch.randn(hd, generator=g) for _ in range(4))
    out, mean, rstd = torch_ops.qk_norm_fwd(qkv, H, hd, wq, bq, wk, bk, 1e-5)

    x = qkv.double().requires_grad_(True)
    pw = [t.double().requires_grad_(True) for t in (wq, bq, wk, bk)]
    q = F.layer_norm(x[:, :D].view(T, H, hd), (hd,), pw[0], pw[1], 1e-5)
    k = F.layer_norm(x[:, D:2 * D].view(T, H, hd), (hd,), pw[2], pw[3], 1e-5)
    ref = torch.cat([q.reshape(T, D), k.reshape(T, D), x[:, 2 * D:]], dim=1)
    assert _rel(out, ref) < 1e-5
    assert out.data_ptr() != qkv.data_ptr() and torch.equal(out[:, 2 * D:], qkv[:, 2 * D:])
    xs = qkv[:, :2 * D].double().reshape(T, 2, H, hd)
    assert _rel(mean.view(T, 2, H), xs.mean(-1)) < 1e-6
    assert _rel(rstd.view(T, 2, H), torch.rsqrt(xs.var(-1, unbiased=False) + 1e-5)) < 1e-5

    dout = torch.randn(T, 3 * D, generator=g)
    ref.backward(dout.double())
    dqkv = dout.clone()
    res, dwq, dbq, dwk, dbk, cs = torch_ops.qk_norm_bwd(dqkv, qkv, H, hd, wq, wk, mean, rstd)
    assert res is dqkv
    assert _rel(dqkv[:, :2 * D], x.grad[:, :2 * D]) < 1e-5
    assert torch.equal(dqkv[:, 2 * D:], dout[:, 2 * D:])  # dv untouched
    for got, want in zip((dwq, dbq, dwk, dbk), pw):
        assert _rel(got, want.grad) < 1e-5
    assert _rel(cs, x.grad[:, :2 * D].sum(0)) < 1e-5

    # in place: the same values, v untouched, and the same buffer
    buf = qkv.clone()
    out2, _, _ = torch_ops.qk_norm_fwd(buf, H, hd, wq, bq, wk, bk, 1e-5, inplace=True)
    assert out2 is buf and torch.equal(out2, out)


def test_column_sums_are_those_of_the_stored_gradient():
    """colsum is the sum of the dq / dk that were stored (rounded to the buffer's dtype), not of the fp32 values."""
    g = torch.Generator().manual_seed(1)
    T, H, hd = 33, 2, 16
    qkv = torch.randn(T, 3 * H * hd, generator=g).to(torch.bfloat16)
    w = [torch.randn(hd, generator=g).to(torch.bfloat16) for _ in range(4)]
    _, mean, rstd = torch_ops.qk_norm_fwd(qkv, H, hd, *w, 1e-5)
    dqkv = torch.randn(T, 3 * H * hd, generator=g).to(torch.bfloat16)
    *_, cs = torch_ops.qk_norm_bwd(dqkv, qkv, H, hd, w[0], w[2], mean, rstd)
    assert dqkv.dtype == torch.bfloat16 and cs.dtype == torch.float32
    assert torch.equal(cs, dqkv[:, : 2 * H * hd].float().sum(0))


# ------------------------------------------------------------------------------------------------
# the engine against the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grad_ckpt,keep,flatten", [(True, 0, False), (False, 0, False), (True, 0, True),
                                                    (False, 0, True), (True, 1, False), (True, 99, False)])
def test_engine_matches_autograd(grad_ckpt, keep, flatten):
    torch.manual_seed(0)
    cfg = qk_cfg()
    model = FSDPViT(cfg, dtype=torch.float32, grad_ckpt=grad_ckpt, ckpt_keep_blocks=keep, flatten_parameters=flatten,
                    seed=3)
    randomize_qk_params(model)
    images = torch.randn(4, 3, cfg.image_size, cfg.image_size)
    ref_logits = _check_against_oracle(model, images, TARGET)
    assert torch.allclose(model.eval()(images).double(), ref_logits.detach(), atol=1e-4)


@pytest.mark.parametrize("extras", [{"P": 99, "h": 99, "g": 99}, {"P": 1, "h": 0, "g": 1}, {"P": 0, "h": 99, "g": 0}])
def test_kept_blocks_with_extras_match_autograd(extras):
    torch.manual_seed(0)
    model = FSDPViT(qk_cfg(), dtype=torch.float32, grad_ckpt=True, ckpt_keep_blocks=99, seed=3)
    model.keep_extras = extras
    randomize_qk_params(model, seed=1)
    _check_against_oracle(model, IMAGES, TARGET)


def test_flash_style_path_matches_autograd(monkeypatch):
    monkeypatch.setattr(torch_ops, "FLASH_ATTENTION", True)
    for kw in (dict(ckpt_keep_blocks=0), dict(ckpt_keep_blocks=99), dict(grad_ckpt=False)):
        model = FSDPViT(qk_cfg(), dtype=torch.float32, seed=3, **kw)
        randomize_qk_params(model, seed=2)
        _check_against_oracle(model, IMAGES, TARGET)


def _model_masks(model, B):
    """The multiplicative dropout / drop-path factors the model's blocks draw in its next training step (the masks of
    torch_ops.dropout and torch_ops.drop_path_scale for the keys of vit.block_forward)."""
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
    cfg = qk_cfg(num_blocks=4, **kw)
    model = FSDPViT(cfg, dtype=torch.float32, seed=3, **mode)
    randomize_qk_params(model, seed=3)
    images = torch.randn(8, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(2))
    target = torch.randint(0, 10, (8,), generator=torch.Generator().manual_seed(2))
    masks = _model_masks(model, 8)
    _check_against_oracle(model, images, target, masks)


# ------------------------------------------------------------------------------------------------
# default behaviour, parameters, config
# ------------------------------------------------------------------------------------------------
def test_flag_off_calls_nothing_new(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("qk_norm op called without --qk_norm")

    monkeypatch.setattr(torch_ops, "qk_norm_fwd", boom)
    monkeypatch.setattr(torch_ops, "qk_norm_bwd", boom)
    for kw in (dict(grad_ckpt=True), dict(grad_ckpt=False), dict(grad_ckpt=True, ckpt_keep_blocks=2)):
        FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3, **kw).forward_backward(IMAGES, TARGET)
    assert not any("_norm." in n for n, _ in vit.block_param_specs(tiny_cfg()))
    assert set(vit.init_block_params(tiny_cfg(), torch.Generator().manual_seed(0))) == {
        n for n, _ in vit.block_param_specs(tiny_cfg())}


def test_parameters_order_init_and_count():
    cfg = qk_cfg()
    names = [n for n, _ in vit.block_param_specs(cfg)]
    i = names.index("attn.qkv.bias")
    assert names[i + 1: i + 5] == ["attn.q_norm.weight", "attn.q_norm.bias", "attn.k_norm.weight", "attn.k_norm.bias"]
    assert all(s == (cfg.head_dim,) for n, s in vit.block_param_specs(cfg) if "_norm." in n)
    a = full_params_of(FSDPViT(cfg, dtype=torch.float32, seed=5))
    b = full_params_of(FSDPViT(tiny_cfg(), dtype=torch.float32, seed=5))
    for k, v in a.items():
        if ".q_norm." in k or ".k_norm." in k:
            assert torch.equal(v, torch.ones_like(v) if k.endswith("weight") else torch.zeros_like(v)), k
        else:
            assert torch.equal(v, b[k]), k  # the norms draw nothing: every other parameter is the same-seed one
    assert set(a) - set(b) == {f"blocks.{i}.attn.{n}.{p}" for i in range(cfg.num_blocks) for n in ("q_norm", "k_norm")
                               for p in ("weight", "bias")}
    assert cfg.block_numel() == tiny_cfg().block_numel() + 4 * cfg.head_dim
    assert cfg.block_numel() == sum(torch.Size(s).numel() for _, s in vit.block_param_specs(cfg))
    big = ViTConfig(qk_norm=True)
    assert big.block_numel() - ViTConfig().block_numel() == 4 * 160
    assert big.flops_per_image() == ViTConfig().flops_per_image()


def test_loss_differs_from_the_model_without_the_flag():
    a = FSDPViT(qk_cfg(), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    assert abs(a.forward_backward(IMAGES, TARGET).item() - b.forward_backward(IMAGES, TARGET).item()) > 1e-4


def test_lean_bytes_count_the_statistics():
    a = FSDPViT(qk_cfg(), dtype=torch.float32, seed=3)
    b = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    cfg = a.cfg
    assert a.lean_bytes_per_block(4) - b.lean_bytes_per_block(4) == 16 * 4 * cfg.num_patches * cfg.num_heads


def test_cli_parsing():
    assert parse_args([]).qk_norm is False
    assert ViTConfig.from_args(parse_args([])).qk_norm is False
    args = parse_args(["--qk_norm"])
    assert args.qk_norm is True and ViTConfig.from_args(args).qk_norm is True


def test_cuda_graph_accepts_qk_norm_checks():
    """The norm takes no host values: the graph wrapper's refusals do not mention it (CPU models are refused for being
    on the CPU, not for --qk_norm)."""
    model = FSDPViT(qk_cfg(), dtype=torch.float32, seed=3)
    with pytest.raises(RuntimeError, match="CUDA model"):
        GraphedTrainStep(model, ShardedAdamW(model, lr=1e-3))


# ------------------------------------------------------------------------------------------------
# FSDP equivalence and checkpoints
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def qk_baseline(tmp_path_factory):
    out = tmp_path_factory.mktemp("qk_base") / "r.json"
    return launch(1, {"model": {"qk_norm": True}, "steps": 4}, str(out))


def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.mark.parametrize("opts", [{}, {"flatten": True}])
def test_two_ranks_reproduce_one(opts, qk_baseline, tmp_path):
    res = launch(2, dict(opts, model={"qk_norm": True}, steps=4), str(tmp_path / "r.json"))
    _close(res["losses"], qk_baseline["losses"])
    _close(res["norms"], qk_baseline["norms"], tol=1e-4)


def test_resume_equals_uninterrupted(tmp_path, qk_baseline):
    d = str(tmp_path)
    model = {"qk_norm": True}
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
    # two training steps so that the norms' parameters are no longer ones / zeros
    launch(2, {"model": {"qk_norm": True}, "steps": 2, "seed": 7, "dump_state": prefix + "_rank_{rank}.ckpt"},
           os.path.join(d, "r.json"))
    full = consolidate_files(prefix, save_path=prefix + "_full.pth")
    assert full["blocks.0.attn.q_norm.weight"].shape == (qk_cfg().head_dim,)
    assert not torch.equal(full["blocks.0.attn.q_norm.weight"], torch.ones(qk_cfg().head_dim))
    cfg = qk_cfg()
    engine = FSDPViT(cfg, dtype=torch.float32, seed=99)
    engine.load_full_state_dict(full)
    plain = PlainViT.from_consolidated(prefix + "_full.pth", cfg).eval()
    assert set(plain.state_dict()) == set(full)
    images = torch.randn(3, 3, cfg.image_size, cfg.image_size)
    with torch.no_grad():
        want = plain(images)
    got = engine.eval()(images)
    assert torch.allclose(got, want, atol=1e-4), (got - want).abs().max()


def test_full_checkpoint_refusals():
    with_qk = full_params_of(FSDPViT(qk_cfg(), dtype=torch.float32, seed=1))
    without = full_params_of(FSDPViT(tiny_cfg(), dtype=torch.float32, seed=1))
    with pytest.raises(ValueError, match="uses --qk_norm, but the checkpoint has no attn.q_norm"):
        FSDPViT(qk_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(without)
    with pytest.raises(ValueError, match="pass --qk_norm to load it"):
        FSDPViT(tiny_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(with_qk)
    FSDPViT(qk_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(with_qk)  # the matching pairs load
    FSDPViT(tiny_cfg(), dtype=torch.float32, seed=2).load_full_state_dict(without)


def test_full_checkpoint_refusal_through_the_cli(tmp_path):
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    full = str(tmp_path / "plain.pth")
    sd = full_params_of(FSDPViT(tiny_cfg(num_blocks=2, embed_dim=32, num_heads=2), dtype=torch.float32, seed=1))
    sd["pos_embed"] = sd["pos_embed"][None]  # the consolidated (timm) shape [1, N, D]
    torch.save({"model": sd}, full)
    args = ["run_vit_training.py", "--fake_data", "--device", "cpu", "--nproc", "1", "--image_size", "32",
            "--patch_size", "8", "--embed_dim", "32", "--num_heads", "2", "--num_blocks", "2", "--mlp_ratio", "2",
            "--num_classes", "10", "--batch_size", "4", "--max_steps", "1", "--num_workers", "0", "--num_epochs", "1",
            "--ckpt_dir", str(tmp_path / "c"), "--init_from_full_ckpt", full, "--qk_norm"]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, *args], cwd=root, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode != 0
    assert "uses --qk_norm, but the checkpoint has no attn.q_norm" in r.stdout + r.stderr


# ------------------------------------------------------------------------------------------------
# build: the new kernels compile for sm_90a without spills or calls
# ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")),
                    reason="needs nvcc")
def test_qk_norm_kernels_compile_for_sm90a_without_spills(tmp_path):
    from vit_10b_fsdp_example_b200 import build_ext

    nvcc = os.path.join(build_ext._cuda_home(), "bin", "nvcc")
    res = subprocess.run([nvcc, *build_ext.NVCC_FLAGS, "-Xptxas", "-v", "-I", build_ext.CSRC, "-c",
                          os.path.join(build_ext.CSRC, "qk_norm.cu"), "-o", str(tmp_path / "q.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = (res.stdout + res.stderr).splitlines()
    found = {}
    for i, ln in enumerate(lines):
        if "Compiling entry function" in ln:
            assert "sm_90a" in ln
            found[ln.split("'")[1]] = next(x for x in lines[i + 1:] if "spill stores" in x)
    assert sum("qk_norm_fwd_kernel" in k for k in found) == 4 and sum("qk_norm_bwd_kernel" in k for k in found) == 3
    assert all("0 bytes spill stores, 0 bytes spill loads" in v for v in found.values()), found
    if shutil.which("cuobjdump"):
        sass = subprocess.run(["cuobjdump", "-sass", str(tmp_path / "q.o")], capture_output=True, text=True).stdout
        assert "qk_norm_bwd_kernel" in sass and " CALL" not in sass
