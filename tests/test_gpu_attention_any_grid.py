"""Patch grids whose token count N the fused attention pair does not take: odd N (ViT-B/32 at 224 px: 49 tokens, 240 px
at patch 16: 225, 518 px at patch 14: 1369) and long even N at head dims that are not routed (ViT-H/14 at 476 px: 1156
tokens at hd 80).  They run the un-fused route: batched wgmma GEMMs with P materialised as [B*H, N, pad8(N)] and the
softmax kernels, whose odd / long rows go to the vector kernels."""
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
KEY = 0x5EED_0DD


def _close(got, ref, rel=3e-2, what=""):
    from helpers import assert_close_elementwise

    assert_close_elementwise(got, ref, rtol=rel, atol_rel=rel, what=what)


def _close_max(got, ref, what, rel=3e-2):
    err = (got.float() - ref.float()).abs().max().item() / (ref.float().abs().max().item() + 1e-6)
    assert err < rel, f"{what}: rel err {err}"


def _masked_reference(qkv, dout, B, N, H, hd, keep, scale):
    """fp32 attention forward + backward with the dropout mask `keep` [B, H, N, N] and keep-scale `scale`."""
    D = H * hd
    q, k, v = qkv.float().view(B, N, 3, H, hd).permute(2, 0, 3, 1, 4)
    do = dout.float().view(B, N, H, hd).permute(0, 2, 1, 3)
    p = torch.softmax((q @ k.transpose(-1, -2)) * hd ** -0.5, dim=-1)
    m = keep.float() * scale
    out = ((p * m) @ v).permute(0, 2, 1, 3).reshape(B * N, D)
    dv = (p * m).transpose(-1, -2) @ do
    dpm = (do @ v.transpose(-1, -2)) * m
    ds = hd ** -0.5 * p * (dpm - (dpm * p).sum(-1, keepdim=True))
    dqkv = torch.stack([ds @ k, ds.transpose(-1, -2) @ q, dv], 0).permute(1, 3, 0, 2, 4).reshape(B * N, 3 * D)
    return out, dqkv


@pytest.mark.parametrize("drop", [None, 0.1])
@pytest.mark.parametrize("N,hd", [(49, 64), (225, 40), (1369, 104), (1369, 160), (1156, 80)])
def test_unfused_attention_at_any_grid(N, hd, drop):
    from vit_10b_fsdp_example_b200.ops import cuda_ops as co, torch_ops as to

    assert not co.use_flash(N, hd) and not co._C.attention_supported(N, hd)
    B, H = (2, 3) if N < 1000 else (1, 2)
    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(N * 1000 + hd)
    qkv = (torch.randn(B * N, 3 * D, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    dout = torch.randn(B * N, D, device="cuda", generator=g).to(torch.bfloat16)
    dr = None if drop is None else (drop, KEY)
    out, p = co.attention_fwd(qkv, B, N, H, hd, drop=dr)
    assert p.shape == (B * H, N, (N + 7) // 8 * 8)
    dqkv, cs = co.attention_bwd(dout, qkv, p, B, N, H, hd, want_colsum=True, drop=dr)
    if drop is None:
        outr, pr = to.attention_fwd(qkv.float(), B, N, H, hd)
        _close(p[..., :N].reshape(B, H, N, N), pr, what="P")
        dqkvr = to.attention_bwd(dout.float(), qkv.float(), pr, B, N, H, hd)
    else:
        ldp = (N + 7) // 8 * 8
        ones = torch.ones(B * H, N, ldp, device="cuda", dtype=torch.bfloat16)
        kept = co.dropout(ones, drop, KEY)[..., :N].reshape(B, H, N, N)
        keep = kept != 0
        assert 0.85 < keep.float().mean().item() < 0.95
        scale = 1.0 / (1.0 - int(drop * 65536.0 + 0.5) / 65536.0)  # the kernels' keep-scale, before bf16 rounding
        outr, dqkvr = _masked_reference(qkv, dout, B, N, H, hd, keep, scale)
    _close(out, outr, what="out")
    for name, i in (("dq", 0), ("dk", 1), ("dv", 2)):
        sl = slice(i * D, (i + 1) * D)
        _close_max(dqkv[:, sl], dqkvr[:, sl], name)
    csr = dqkv.float().sum(dim=0)  # the qkv bias gradient: column sums of the bf16 values that were stored
    assert (cs - csr).abs().max().item() <= 2e-3 * csr.abs().max().item() + 1e-3, "qkv bias gradient"
    _close_max(cs, dqkvr.float().sum(dim=0), "qkv bias gradient vs fp32", rel=5e-2)


def _full_grads(model):
    return {u.name: u.shard_grad.float().clone() for u in model.all_units}


@pytest.mark.parametrize("image_size,patch_size,dim", [(224, 32, 128), (70, 14, 160)])
def test_engine_at_odd_grid_matches_the_cpu_path(image_size, patch_size, dim):
    """49 and 25 tokens: the bf16 GPU model matches the fp32 CPU model (same seed) in loss and gradients, with every
    block recomputing P in backward (ckpt_keep_blocks 0) and with both blocks keeping it (2)."""
    from vit_10b_fsdp_example_b200.config import ViTConfig
    from vit_10b_fsdp_example_b200.parallel import FSDPViT

    cfg = ViTConfig(image_size=image_size, patch_size=patch_size, embed_dim=dim, num_heads=2, num_blocks=2,
                    mlp_ratio=4.0, num_classes=96)
    assert cfg.num_patches % 2 == 1
    g = torch.Generator().manual_seed(0)
    x = torch.randn(4, 3, image_size, image_size, generator=g)
    y = torch.randint(0, 96, (4,), generator=g)
    for keep in (0, 2):
        res = []
        for dev, dtype in ((torch.device("cpu"), torch.float32), (torch.device("cuda"), torch.bfloat16)):
            model = FSDPViT(cfg, device=dev, dtype=dtype, seed=4, ckpt_keep_blocks=keep)
            loss = model.forward_backward(x.to(dev), y.to(dev)).item()
            res.append((loss, _full_grads(model)))
        (loss_ref, g_ref), (loss, grads) = res
        assert math.isfinite(loss) and abs(loss - loss_ref) < 1e-2 * abs(loss_ref) + 1e-2, (keep, loss, loss_ref)
        for k in g_ref:
            a, b = g_ref[k], grads[k].cpu()
            assert (a - b).norm().item() <= 5e-2 * a.norm().item() + 1e-6, (keep, k)


def test_cli_trains_at_patch_32(tmp_path):
    """run_vit_training.py on the GPU at 224 px / patch 32 (7 x 7 tokens): two steps of a small model."""
    args = ["--fake_data", "--device", "cuda", "--nproc", "1", "--image_size", "224", "--patch_size", "32",
            "--embed_dim", "128", "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8",
            "--warmup_steps", "2", "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0",
            "--num_epochs", "1", "--ckpt_epoch_interval", "100", "--test_epoch_interval", "100"]
    r = subprocess.run([sys.executable, "run_vit_training.py", *args, "--ckpt_dir", str(tmp_path)], cwd=ROOT,
                       env=dict(os.environ, MASTER_ADDR="127.0.0.1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    losses = [float(v) for v in re.findall(r"loss: ([0-9.eE+-]+|nan|inf)", r.stdout)]
    assert len(losses) == 2 and all(math.isfinite(v) for v in losses), r.stdout[-2000:]
