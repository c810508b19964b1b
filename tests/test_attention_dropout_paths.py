"""Attention dropout on the fused (flash-style) attention path: the CPU model path against the un-fused one, and the
compiled dropout instantiations of the fused kernels (cuobjdump -sass of the in-tree build, CPU only)."""
import os
import shutil
import sys

import pytest
import torch

from helpers import full_grads_of, tiny_cfg
from vit_10b_fsdp_example_b200.parallel import FSDPViT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "vit_10b_fsdp_example_b200", "csrc", "build")


def test_flash_dropout_path_matches_unfused_on_cpu(monkeypatch):
    """Same [B, H, N, N] mask shape on both routes -> same CPU mask: gradients with the lse pair and dropout match the
    un-fused route that drops the materialised P; checkpointed, non-checkpointed and kept blocks agree too."""
    from vit_10b_fsdp_example_b200.ops import torch_ops

    cfg = tiny_cfg(att_dropout=0.2)
    images = torch.randn(4, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(0))
    target = torch.tensor([1, 5, 7, 2])
    runs = []
    for flash, ckpt, keep in ((False, True, 0), (True, True, 0), (True, False, 0), (True, True, 1)):
        monkeypatch.setattr(torch_ops, "FLASH_ATTENTION", flash)
        model = FSDPViT(cfg, dtype=torch.float32, grad_ckpt=ckpt, ckpt_keep_blocks=keep, seed=3)
        loss = model.forward_backward(images, target).item()
        runs.append((loss, full_grads_of(model)))
    (loss0, g0), rest = runs[0], runs[1:]
    for loss, g in rest:
        assert abs(loss - loss0) < 1e-5
        for k in g0:
            assert (g[k] - g0[k]).abs().max().item() <= 2e-4 * g0[k].abs().max().item() + 1e-7, k
    # dropout really is on: without it the gradients differ
    monkeypatch.setattr(torch_ops, "FLASH_ATTENTION", True)
    model = FSDPViT(tiny_cfg(), dtype=torch.float32, seed=3)
    model.forward_backward(images, target)
    plain = full_grads_of(model)
    assert any((plain[k] - g0[k]).abs().max().item() > 1e-4 for k in g0)


@pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(os.path.join(BUILD, "attention_drop_sm90.cu.o")),
                    reason="needs cuobjdump and the in-tree build (python -m vit_10b_fsdp_example_b200.build_ext)")
def test_dropout_attention_kernels_are_call_free_wgmma_tma_kernels():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_summary
    import subprocess

    census = sass_summary.census(BUILD, ["attention_drop_sm90.cu.o"])["attention_drop_sm90.cu.o"]
    txt = subprocess.run(["cuobjdump", "-sass", os.path.join(BUILD, "attention_drop_sm90.cu.o")], capture_output=True,
                         text=True).stdout
    names = [f"attn_fwd_drop_sm90_kernel<{hd}>" for hd in (64, 128, 160)] + \
            [f"attn_bwd_drop_sm90_kernel<{hd}, {r}>" for hd in (64, 128, 160) for r in (0, 1)]
    for name in names:
        kernels = {k: c for k, c in census.items() if k.endswith(name)}
        assert len(kernels) == 1, name
        for c in kernels.values():
            for prefix in ("HGMMA.64", "UTMALDG.4D", "SYNCS.PHASECHK"):
                assert any(op.startswith(prefix) for op in c), (name, prefix)
    # no CALL anywhere in the object: a call would make ptxas serialise the wgmma batches
    assert " CALL" not in txt
