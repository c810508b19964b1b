"""Per-rank sharded checkpoints (reference: utils.py:24-43, run_vit_training.py:245-248,297-299).

Layout kept compatible with the reference: one ``torch.save`` file per rank per epoch named
``epoch_{E}_rank_{R}.ckpt`` holding exactly four keys -- ``model`` (this rank's shards), ``shard_metadata``
(``None`` when not FSDP), ``optimizer`` and ``lr_scheduler`` -- plus a fifth, ``model_ema`` (this rank's EMA shards,
same layout as ``model``), only when the model keeps an EMA (``--model_ema``), and a sixth, ``rope`` (the
``rope`` / ``rope_theta`` / ``rope_ref_grid`` settings), only with ``--rope``: the rotary embedding has no parameters,
so only this record tells a resumed run how the weights were trained; a checkpoint without it had no RoPE.  Every rank writes its own file; loading
goes through the host (``map_location='cpu'``).  ``consolidate_sharded_ckpts`` rebuilds a full state_dict.
"""
from __future__ import annotations

import math
import os

import torch


def save_ckpt(ckpt_path: str, model, optimizer, lr_scheduler, master_only: bool = True, rank: int = 0,
              barrier=None) -> None:
    ckpt = {
        "model": model.state_dict(),
        "shard_metadata": model.get_shard_metadata() if getattr(model, "use_fsdp", False) else None,
        "optimizer": optimizer.state_dict(),
        "lr_scheduler": lr_scheduler.state_dict(),
    }
    if getattr(model, "has_ema", False):
        ckpt["model_ema"] = model.ema_state_dict()
    rope = rope_settings(getattr(model, "cfg", None))
    if rope is not None:
        ckpt["rope"] = rope
    if not master_only or rank == 0:
        os.makedirs(os.path.dirname(os.path.abspath(ckpt_path)), exist_ok=True)
        tmp = ckpt_path + ".tmp"
        torch.save(ckpt, tmp)
        os.replace(tmp, ckpt_path)  # never leave a half-written checkpoint behind
    if barrier is not None:
        barrier()  # xm.save contains a rendezvous
    print(f"checkpoint saved to {ckpt_path}\n", end="")


def rope_settings(cfg):
    """The RoPE record of a checkpoint: {"rope": True, "rope_theta": .., "rope_ref_grid": ..}, or None without RoPE."""
    if cfg is None or not getattr(cfg, "rope", False):
        return None
    return {"rope": True, "rope_theta": float(cfg.rope_theta), "rope_ref_grid": int(cfg.rope_ref_grid)}


def check_rope_settings(saved, cfg, ckpt_path: str) -> None:
    """Refuses to resume weights trained under other RoPE settings, naming the flags that would match them."""
    want = rope_settings(cfg)
    if saved == want:
        return
    if saved is None:
        fix = "drop --rope, --rope_theta and --rope_ref_grid"
    else:
        fix = f"pass --rope --rope_theta {saved['rope_theta']:g} --rope_ref_grid {saved['rope_ref_grid']}"
    raise ValueError(f"checkpoint {ckpt_path} was trained with rotary position embedding settings {saved or 'no RoPE'}, "
                     f"this run has {want or 'no RoPE'}: {fix} to resume it")


def load_ckpt(ckpt_path: str, model, optimizer, lr_scheduler) -> None:
    assert os.path.exists(ckpt_path), f"checkpoint {ckpt_path} does not exist"
    ckpt = torch.load(ckpt_path, map_location="cpu", weights_only=False)
    if hasattr(model, "cfg"):
        check_rope_settings(ckpt.get("rope"), model.cfg, ckpt_path)
    try:
        model.load_state_dict(ckpt["model"], shard_metadata=ckpt.get("shard_metadata"))
    except TypeError:  # a plain nn.Module-style model
        model.load_state_dict(ckpt["model"])
    if getattr(model, "has_ema", False):  # a model_ema in a checkpoint is ignored when the model keeps no EMA
        if "model_ema" in ckpt:
            model.load_ema_state_dict(ckpt["model_ema"])
        else:
            model.reset_ema()
            print("the checkpoint has no model_ema: the model EMA starts from the restored weights\n", end="")
    optimizer.load_state_dict(ckpt["optimizer"])
    if getattr(model, "step_count", None) == 0 and hasattr(optimizer, "state") and hasattr(model, "all_units"):
        # DDP checkpoints carry no shard metadata: the optimizer step count is the number of steps taken
        model.step_count = int(optimizer.state[model.all_units[0].name]["step"])
    lr_scheduler.load_state_dict(ckpt["lr_scheduler"])
    print(f"resumed from checkpoint {ckpt_path}\n", end="")


def resize_pos_embed(pos_embed: torch.Tensor, num_patches: int, embed_dim: int,
                     num_prefix_tokens: int = 0) -> torch.Tensor:
    """Resample a checkpoint's ``pos_embed`` [1, P + g0*g0, D] to the model's [1, P + num_patches, D], for fine-tuning
    at another image size: the first P = ``num_prefix_tokens`` rows (class / register tokens) pass through unchanged and
    the grid rows are resampled bicubically, ``align_corners=False``, in fp32 over the [g0, g0, D] grid (timm's
    ``resize_pos_embed`` with ``num_tokens``; later timm releases call it ``resample_abs_pos_embed`` and antialias by
    default, which this does not).  Returns ``pos_embed`` itself when the grids match."""
    if pos_embed.dim() != 3 or pos_embed.shape[0] != 1:
        raise ValueError(f"pos_embed: expected shape [1, N, D], got {tuple(pos_embed.shape)}")
    P = num_prefix_tokens
    n0, d0 = pos_embed.shape[1] - P, pos_embed.shape[2]
    if d0 != embed_dim:
        raise ValueError(f"pos_embed: checkpoint embed dim {d0} does not match the model's {embed_dim}")
    if n0 == num_patches:
        return pos_embed
    g0, g = math.isqrt(max(n0, 0)), math.isqrt(num_patches)
    if n0 < 1 or g0 * g0 != n0 or g * g != num_patches:
        after = f" after its {P} prefix rows" if P else ""
        raise ValueError(f"pos_embed: cannot resample {n0} to {num_patches} tokens{after}: both must be square grids")
    grid = pos_embed[:, P:].detach().float().reshape(1, g0, g0, d0).permute(0, 3, 1, 2)
    grid = torch.nn.functional.interpolate(grid, size=(g, g), mode="bicubic", align_corners=False)
    grid = grid.permute(0, 2, 3, 1).reshape(1, num_patches, d0).to(pos_embed.dtype)
    return torch.cat([pos_embed[:, :P].detach(), grid], dim=1) if P else grid


_WRAPPER_PARTS =("_fsdp_wrapped_module.", "_fpw_module.", "_checkpoint_wrapped_module.", "_orig_mod.")


def normalize_full_state_dict_keys(state: dict) -> dict:
    """Strip wrapper prefixes from the parameter names of a consolidated checkpoint so that one written by another
    stack loads here: torch_xla FSDP (``_fsdp_wrapped_module.`` / ``_fpw_module.``, what the reference's
    ``consolidate_sharded_ckpts`` may leave behind), PyTorch FSDP / activation-checkpoint wrappers, DDP's leading
    ``module.`` and torch.compile's ``_orig_mod.``.  Names that are already timm-style pass through unchanged."""
    out = {}
    for k, v in state.items():
        name = k
        for part in _WRAPPER_PARTS:
            name = name.replace(part, "")
        while name.startswith("module."):
            name = name[len("module."):]
        if name in out:
            raise KeyError(f"checkpoint keys {k!r} and another entry both normalise to {name!r}")
        out[name] = v
    return out
