"""Fine-tuning at another resolution: --init_from_full_ckpt resamples a checkpoint's pos_embed to the model's patch grid
(utils/checkpoint.resize_pos_embed: bicubic, align_corners=False, fp32, over the [g, g, D] grid)."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from vit_10b_fsdp_example_b200.utils.checkpoint import resize_pos_embed  # noqa: E402


@pytest.mark.parametrize("g0,g,dtype", [(16, 37, torch.float32), (2, 3, torch.float32), (16, 37, torch.bfloat16)])
def test_matches_bicubic_interpolation_of_the_grid(g0, g, dtype):
    D = 24
    pe = torch.randn(1, g0 * g0, D, generator=torch.Generator().manual_seed(g0)).to(dtype)
    out = resize_pos_embed(pe, g * g, D)
    grid = pe.float().reshape(1, g0, g0, D).permute(0, 3, 1, 2)
    ref = F.interpolate(grid, size=(g, g), mode="bicubic", align_corners=False).permute(0, 2, 3, 1).reshape(1, g * g, D)
    assert out.shape == (1, g * g, D) and out.dtype == dtype
    assert torch.equal(out, ref.to(dtype))
    # token (row r, column c) of the grid is pos_embed[0, r * g + c]: a ramp along the columns stays one
    ramp = torch.arange(g0, dtype=torch.float32).repeat(g0).view(1, g0 * g0, 1).expand(1, g0 * g0, D)
    out = resize_pos_embed(ramp, g * g, D).view(g, g, D)
    assert torch.allclose(out[0], out[-1]) and not torch.allclose(out[:, 0], out[:, -1])


def test_equal_grids_return_the_tensor_unchanged():
    pe = torch.randn(1, 49, 16)
    assert resize_pos_embed(pe, 49, 16) is pe


@pytest.mark.parametrize("shape,n,d,msg", [((1, 49, 16), 64, 32, "embed dim 16"),
                                          ((1, 48, 16), 64, 16, "square"),
                                          ((1, 49, 16), 50, 16, "square"),
                                          ((49, 16), 64, 16, r"\[1, N, D\]")])
def test_rejects_what_cannot_be_resampled(shape, n, d, msg):
    with pytest.raises(ValueError, match=msg):
        resize_pos_embed(torch.zeros(shape), n, d)


def _run(args):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, *args], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def _consolidate(ckpt_dir, path):
    _run(["-m", "vit_10b_fsdp_example_b200.consolidate_sharded_ckpts", "--ckpt_prefix",
          os.path.join(ckpt_dir, "epoch_1"), "--save_path", path])
    sd = torch.load(path, map_location="cpu", weights_only=False)
    return sd.get("model", sd)


def test_init_from_a_checkpoint_at_another_image_size_via_cli(tmp_path):
    """Train at 28 px / patch 14 (2 x 2 tokens), consolidate, start a run at 42 px (3 x 3 tokens, an odd count) from it
    with the learning rate at 0: its pos_embed is the resampled one."""
    common = ["--fake_data", "--device", "cpu", "--nproc", "1", "--patch_size", "14", "--embed_dim", "32",
              "--num_heads", "2", "--num_blocks", "1", "--num_classes", "10", "--batch_size", "4", "--warmup_steps", "1",
              "--max_steps", "2", "--log_step_interval", "1", "--num_workers", "0", "--num_epochs", "1",
              "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1"]
    _run(["run_vit_training.py", *common, "--image_size", "28", "--ckpt_dir", str(tmp_path / "a")])
    full = _consolidate(str(tmp_path / "a"), str(tmp_path / "a.pth"))
    assert full["pos_embed"].shape == (1, 4, 32)

    out = _run(["run_vit_training.py", *common, "--image_size", "42", "--lr", "0", "--weight_decay", "0",
                "--init_from_full_ckpt", str(tmp_path / "a.pth"), "--ckpt_dir", str(tmp_path / "b")])
    assert out.count("pos_embed resampled from 4 to 9 tokens") == 1
    new = _consolidate(str(tmp_path / "b"), str(tmp_path / "b.pth"))
    want = resize_pos_embed(full["pos_embed"], 9, 32)
    assert new["pos_embed"].shape == (1, 9, 32)
    assert torch.equal(new["pos_embed"].float(), want.float())
    assert torch.equal(new["blocks.0.attn.qkv.weight"].float(), full["blocks.0.attn.qkv.weight"].float())
