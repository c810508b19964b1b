"""Offline consolidation of per-rank sharded checkpoints into one full ``state_dict``.

Equivalent of ``python3 -m torch_xla.distributed.fsdp.consolidate_sharded_ckpts`` that the reference's
checkpoint layout exists to serve (utils.py:27-28):

    python -m vit_10b_fsdp_example_b200.consolidate_sharded_ckpts \
        --ckpt_prefix /tmp/vit_fsdp/epoch_10 --save_path /tmp/vit_fsdp/epoch_10_full.pth

reads ``{prefix}_rank_{0..W-1}.ckpt``, concatenates every group's shards, strips the padding, reshapes to the
parameter shapes (un-flattening flat parameters) and writes a timm-style state_dict
(``pos_embed`` [1,N,D], ``patch_embed.proj.weight`` [D,3,P,P], ``blocks.{i}.attn.qkv.weight`` ...).  When the
shards carry a model EMA (``--model_ema``) it is consolidated the same way and written as ``model_ema`` next to
``model`` (the key DeiT uses).
"""
from __future__ import annotations

import argparse
import os
from typing import Dict, List

import torch

from .parallel.layout import UnitLayout


def consolidate(ckpts: List[dict], key: str = "model") -> Dict[str, torch.Tensor]:
    """The full state_dict of the rank files' ``key`` entry: ``model``, or ``model_ema`` for the EMA."""
    md0 = ckpts[0]["shard_metadata"]
    assert md0 is not None, "checkpoint was not written by an FSDP model (shard_metadata is None)"
    world = md0["world_size"]
    assert len(ckpts) == world, f"expected {world} rank files, got {len(ckpts)}"
    by_rank = {c["shard_metadata"]["rank"]: c for c in ckpts}
    assert sorted(by_rank) == list(range(world)), "rank files are not a complete 0..W-1 set"
    logical = {k: tuple(v) for k, v in md0.get("logical_shapes", {}).items()}
    patch_k = md0.get("patch_k")
    full_sd: Dict[str, torch.Tensor] = {}
    for umd in md0["units"]:
        lay = UnitLayout.from_metadata(umd)
        full = torch.zeros(lay.full_numel, dtype=torch.float32)
        for r in range(world):
            sd = by_rank[r][key]
            for g in lay.groups:
                piece = sd[f"{lay.name}.{g.name}"]
                off = g.full_offset + r * g.shard_len
                full[off: off + g.shard_len].copy_(piece)
        prefix = "" if lay.name == "root" else lay.name + "."
        for p in lay.params:
            t = full[p.full_offset: p.full_offset + p.numel].view(p.shape).clone()
            if p.name == "patch_embed.proj.weight" and patch_k is not None:
                t = t[:, :patch_k]
            if p.name in logical:
                t = t.reshape(logical[p.name])
            full_sd[prefix + p.name] = t.contiguous()
    return full_sd


def consolidate_files(ckpt_prefix: str, ckpt_suffix: str = "_rank_*.ckpt", save_path: str = "") -> Dict[str, torch.Tensor]:
    import glob

    paths = sorted(glob.glob(ckpt_prefix + ckpt_suffix))
    assert paths, f"no checkpoint files match {ckpt_prefix + ckpt_suffix}"
    # mmap: only the tensors that are actually copied (the model shards) are paged in -- a ViT-10B rank file also
    # carries two fp32 AdamW moments per parameter that consolidation never touches
    ckpts = [torch.load(p, map_location="cpu", weights_only=False, mmap=True) for p in paths]
    full = consolidate(ckpts)
    if save_path:
        out = {"model": full, "shard_metadata": None}
        if all("model_ema" in c for c in ckpts):
            out["model_ema"] = consolidate(ckpts, key="model_ema")
        os.makedirs(os.path.dirname(os.path.abspath(save_path)), exist_ok=True)
        torch.save(out, save_path)
        print(f"consolidated {len(paths)} shard files ({sum(t.numel() for t in full.values()):,} parameters) -> {save_path}")
    return full


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--ckpt_prefix", type=str, required=True, help="e.g. /tmp/vit_fsdp/epoch_10")
    ap.add_argument("--ckpt_suffix", type=str, default="_rank_*.ckpt")
    ap.add_argument("--save_path", type=str, default="")
    args = ap.parse_args(argv)
    save_path = args.save_path or (args.ckpt_prefix + "_consolidated.pth")
    consolidate_files(args.ckpt_prefix, args.ckpt_suffix, save_path)


if __name__ == "__main__":
    main()
