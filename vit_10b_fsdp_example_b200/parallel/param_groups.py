"""Optimizer parameter groups: no weight decay on biases, norms and learned tokens, and layer-wise LR decay.

The rules are MAE's ``param_groups_lrd`` / ``get_layer_id_for_vit`` (also timm's ``create_optimizer_v2`` with
``filter_bias_and_bn=True`` and ``--layer-decay``), applied to the timm parameter names of ``models/vit.py``:

  * no-decay set: every parameter whose *timm* shape (``vit.logical_shapes``, not the stored GEMM shape) has
    ``ndim <= 1``, plus ``pos_embed``, ``cls_token`` and ``reg_token`` (the register tokens are treated exactly like
    the class token).  In a block only ``attn.qkv.weight``, ``attn.proj.weight``, ``mlp.fc1.weight`` and
    ``mlp.fc2.weight`` are decayed; in the root unit only ``patch_embed.proj.weight`` and ``head.weight``.
  * layer ids: ``cls_token``, ``reg_token``, ``pos_embed`` and ``patch_embed.*`` are layer 0, ``blocks.i.*`` is layer
    i + 1, everything else (``norm.*``, ``head.*``) is layer L + 1 with L = num_blocks.  The lr scale of layer ``id`` is
    ``layer_decay ** (L + 1 - id)``: 1 for the head, ``d`` for the last block, ``d ** (L + 1)`` for the stem.

The fused AdamW kernels run over a unit's flat shard, which crosses parameter boundaries, so the groups travel to them
as two small tables per unit (built once, before any CUDA-graph capture):

  * ``chunk_groups``: a uint8 group index for every ``ALIGN`` = 64-element chunk of this rank's shard.  Every parameter
    and every shard group starts at a multiple of 64 elements (``layout.ALIGN``), with or without
    ``--flatten_parameters``, so no chunk holds elements of two parameters; ``build_chunk_groups`` checks that.  A
    padding chunk takes group 0: its gradient and weight are zero, so any group leaves it at zero.
  * ``group_hyper``: fp32 ``[G, 2]`` rows of ``(lr_scale, weight_decay)``, G <= 4 (a block has decay / no-decay, the
    root stem and head x decay / no-decay).

The kernels form each element's ``lr * lr_scale`` and ``1 - lr * lr_scale * wd`` in fp32 from the base lr.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..models import vit
from .layout import ALIGN, UnitLayout

TOKEN_NAMES = ("pos_embed", "cls_token", "reg_token")  # no weight decay, layer 0, whatever their shape


def full_name(unit_name: str, pname: str) -> str:
    """timm name of a unit's parameter: ``blocks.{i}.{pname}`` in a block, ``pname`` in the root unit."""
    return pname if unit_name == "root" else f"{unit_name}.{pname}"


def layer_id(name: str, num_blocks: int) -> int:
    if name in TOKEN_NAMES or name.startswith("patch_embed."):
        return 0
    if name.startswith("blocks."):
        return int(name.split(".")[1]) + 1
    return num_blocks + 1


def decays(name: str, timm_shape: Sequence[int]) -> bool:
    return len(timm_shape) > 1 and name not in TOKEN_NAMES


def lr_scale(lid: int, num_blocks: int, layer_decay: Optional[float]) -> float:
    return 1.0 if layer_decay is None else float(layer_decay) ** (num_blocks + 1 - lid)


def classify(cfg, unit_name: str, specs: Sequence[Tuple[str, Tuple[int, ...]]]) -> Dict[str, Tuple[int, bool]]:
    """pname -> (layer id, decayed?) for the parameters of one unit."""
    logical = vit.logical_shapes(cfg) if unit_name == "root" else {}
    out = {}
    for pname, shape in specs:
        name = full_name(unit_name, pname)
        out[pname] = (layer_id(name, cfg.num_blocks), decays(name, logical.get(pname, shape)))
    return out


def build_chunk_groups(layout: UnitLayout, rank: int, param_group: Dict[str, int]) -> np.ndarray:
    """uint8 group index of every 64-element chunk of `rank`'s shard, from the parameter that owns the chunk."""
    if layout.shard_numel % ALIGN:
        raise AssertionError(f"{layout.name}: shard of {layout.shard_numel} elements is not a multiple of {ALIGN}")
    owner = np.full(layout.shard_numel // ALIGN, -1, dtype=np.int16)
    for g in layout.groups:
        lo_full = g.full_offset + rank * g.shard_len  # the slice of the full buffer this rank owns in shard group g
        if lo_full % ALIGN or g.shard_offset % ALIGN or g.shard_len % ALIGN:
            raise AssertionError(f"{layout.name}/{g.name}: shard group not aligned to {ALIGN} elements")
        for p in layout.params:
            a, b = max(p.full_offset, lo_full), min(p.full_offset + p.numel, lo_full + g.shard_len)
            if a >= b:
                continue
            if p.full_offset % ALIGN:
                raise AssertionError(f"{layout.name}/{p.name}: parameter offset {p.full_offset} is not a multiple of "
                                     f"{ALIGN} elements")
            s = g.shard_offset + (a - lo_full)
            c0, c1 = s // ALIGN, -(-(s + b - a) // ALIGN)
            if (owner[c0:c1] != -1).any():
                raise AssertionError(f"{layout.name}/{p.name}: a {ALIGN}-element chunk of the shard holds two "
                                     f"parameters")
            owner[c0:c1] = param_group[p.name]
    owner[owner < 0] = 0  # padding: gradient and weight are zero, any group leaves it at zero
    return owner.astype(np.uint8)


@dataclass
class GroupRow:
    layer: int
    decay: bool
    lr_scale: float
    weight_decay: float
    tensors: int = 0
    elements: int = 0

    @property
    def name(self) -> str:
        return f"layer_{self.layer}_{'decay' if self.decay else 'no_decay'}"


class UnitGroups:
    """Group tables of one unit on this rank: ``chunk_groups`` (uint8 [shard_numel / 64]) and ``group_hyper``
    (fp32 [G, 2] of (lr_scale, weight_decay)), on the model's device."""

    def __init__(self, rows: List[GroupRow], chunk_groups: torch.Tensor, group_hyper: torch.Tensor):
        self.rows, self.chunk_groups, self.group_hyper = rows, chunk_groups, group_hyper


def build_unit_groups(cfg, layout: UnitLayout, rank: int, weight_decay: float, layer_decay: Optional[float],
                      device) -> UnitGroups:
    specs = [(p.name, p.shape) for p in layout.params]
    cls = classify(cfg, layout.name, specs)
    logical = vit.logical_shapes(cfg) if layout.name == "root" else {}
    keys = sorted(set(cls.values()))
    if len(keys) > 4:
        raise AssertionError(f"{layout.name}: {len(keys)} parameter groups, the kernels' tables hold at most 4")
    rows = [GroupRow(lid, dec, lr_scale(lid, cfg.num_blocks, layer_decay), float(weight_decay) if dec else 0.0)
            for lid, dec in keys]
    index = {k: i for i, k in enumerate(keys)}
    for p in layout.params:
        r = rows[index[cls[p.name]]]
        r.tensors += 1
        r.elements += int(np.prod(logical.get(p.name, p.shape)))  # timm's count (the stored patch weight is padded)
    chunks = build_chunk_groups(layout, rank, {p: index[k] for p, k in cls.items()})
    hyper = torch.tensor([[r.lr_scale, r.weight_decay] for r in rows], dtype=torch.float32)
    return UnitGroups(rows, torch.from_numpy(chunks).to(device), hyper.to(device))


def summary(units: Sequence[UnitGroups]) -> List[GroupRow]:
    """The groups of the whole model, merged over units (timm-style param-group listing)."""
    merged: Dict[Tuple[int, bool], GroupRow] = {}
    for u in units:
        for r in u.rows:
            m = merged.setdefault((r.layer, r.decay), GroupRow(r.layer, r.decay, r.lr_scale, r.weight_decay))
            m.tensors += r.tensors
            m.elements += r.elements
    return [merged[k] for k in sorted(merged)]


def format_summary(rows: Sequence[GroupRow]) -> str:
    return "\n".join(f"{r.name:>20}: lr_scale {r.lr_scale:.6g}, weight_decay {r.weight_decay:g}, "
                     f"{r.tensors} tensors, {r.elements} elements" for r in rows)
