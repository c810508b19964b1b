"""Flat-buffer layout and shard arithmetic of one FSDP unit.

Reference behaviour being reproduced (torch_xla ``XlaFullyShardedDataParallel`` as used at
run_vit_training.py:177-181): every parameter -- or, with ``--flatten_parameters``, one concatenated
flat parameter per unit -- is flattened, zero-padded to a multiple of the world size and chunked; a rank
keeps only its chunk.

H100-first layout: a unit owns ONE contiguous *full* buffer (what the GEMMs read through TMA) and ONE
contiguous *shard* buffer per rank.  The full buffer is a sequence of **shard groups**; group ``g`` spans
``world * g.shard_len`` elements and rank ``r`` owns the r-th ``shard_len`` slice of it:

  flatten_parameters=False : one group per parameter  (per-tensor shards, per-tensor state_dict entries)
  flatten_parameters=True  : one group for the whole unit (a single flat parameter)

Because groups are padded to ``world * shard_len`` the gathered data lands *directly* in its final
position -- an all-gather is ``world`` straight copies per group with no copy-out pass, which is what the
peer-to-peer NVLink kernels exploit.  All offsets are multiples of ALIGN elements (128 B in bf16), so
every parameter view is a legal TMA base address.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

ALIGN = 64  # elements


def ceil_div(a: int, b: int) -> int:
    return -(-a // b)


def round_up(a: int, b: int) -> int:
    return ceil_div(a, b) * b


class ParamViews(dict):
    """name -> parameter view.  ``ag`` optionally maps a weight name to an all-gather-fusion spec: the forward GEMM
    that consumes that weight also pulls its shards from the peers (see Sm100Backend.ag_fuse_spec)."""

    ag: dict = {}

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.ag = {}


@dataclass
class ParamSpec:
    name: str
    shape: Tuple[int, ...]
    numel: int
    full_offset: int  # element offset of the parameter inside the unit's full buffer


@dataclass
class ShardGroup:
    name: str         # parameter name, or "flat_param"
    full_offset: int  # start of the group in the full buffer
    shard_len: int    # elements owned by each rank
    shard_offset: int  # start of this group's slice inside a rank's shard buffer
    numel: int        # un-padded payload elements in the group


@dataclass
class UnitLayout:
    name: str
    world: int
    flatten: bool
    params: List[ParamSpec] = field(default_factory=list)
    groups: List[ShardGroup] = field(default_factory=list)
    full_numel: int = 0
    shard_numel: int = 0

    # -------------------------------------------------------------------------------------------
    @classmethod
    def build(cls, name: str, specs: Sequence[Tuple[str, Tuple[int, ...]]], world: int, flatten: bool) -> "UnitLayout":
        lay = cls(name=name, world=world, flatten=flatten)
        if flatten:
            off = 0
            for pname, shape in specs:
                n = 1
                for d in shape:
                    n *= d
                lay.params.append(ParamSpec(pname, tuple(shape), n, off))
                off = round_up(off + n, ALIGN)
            shard_len = round_up(ceil_div(max(off, 1), world), ALIGN)
            lay.groups.append(ShardGroup("flat_param", 0, shard_len, 0, off))
            lay.full_numel = shard_len * world
            lay.shard_numel = shard_len
        else:
            off = 0
            soff = 0
            for pname, shape in specs:
                n = 1
                for d in shape:
                    n *= d
                shard_len = round_up(ceil_div(n, world), ALIGN)
                lay.params.append(ParamSpec(pname, tuple(shape), n, off))
                lay.groups.append(ShardGroup(pname, off, shard_len, soff, n))
                off += shard_len * world
                soff += shard_len
            lay.full_numel = off
            lay.shard_numel = soff
        return lay

    # -------------------------------------------------------------------------------------------
    def payload_numel(self) -> int:
        return sum(p.numel for p in self.params)

    def param_views(self, full_buf) -> "ParamViews":
        """Name -> shaped view into a full buffer (torch tensor of >= full_numel elements)."""
        return ParamViews({p.name: full_buf[p.full_offset: p.full_offset + p.numel].view(p.shape) for p in self.params})

    def gather_segments(self) -> List[Tuple[int, int, int, int]]:
        """(src_rank, src_shard_offset, dst_full_offset, length) in elements, for every rank."""
        segs = []
        for g in self.groups:
            for r in range(self.world):
                segs.append((r, g.shard_offset, g.full_offset + r * g.shard_len, g.shard_len))
        return segs

    def scatter_segments(self, rank: int) -> List[Tuple[int, int, int]]:
        """(full_offset, shard_offset, length): the slices of a full (gradient) buffer rank owns."""
        return [(g.full_offset + rank * g.shard_len, g.shard_offset, g.shard_len) for g in self.groups]

    def shard_from_full(self, full_buf, rank: int, out):
        """Copy rank's slices of a full buffer into a shard buffer (used at init / load time)."""
        for full_off, shard_off, n in self.scatter_segments(rank):
            out[shard_off: shard_off + n].copy_(full_buf[full_off: full_off + n])
        return out

    def full_from_shards(self, shards, out):
        """Inverse of shard_from_full given all ranks' shard buffers (consolidation / tests)."""
        for r, sh in enumerate(shards):
            for full_off, shard_off, n in self.scatter_segments(r):
                out[full_off: full_off + n].copy_(sh[shard_off: shard_off + n])
        return out

    def metadata(self) -> dict:
        return {
            "name": self.name, "world_size": self.world, "flatten_parameters": self.flatten,
            "full_numel": self.full_numel, "shard_numel": self.shard_numel,
            "params": [{"name": p.name, "shape": list(p.shape), "numel": p.numel, "full_offset": p.full_offset}
                       for p in self.params],
            "groups": [{"name": g.name, "full_offset": g.full_offset, "shard_len": g.shard_len,
                        "shard_offset": g.shard_offset, "numel": g.numel} for g in self.groups],
        }

    @classmethod
    def from_metadata(cls, md: dict) -> "UnitLayout":
        lay = cls(name=md["name"], world=md["world_size"], flatten=md["flatten_parameters"])
        lay.full_numel, lay.shard_numel = md["full_numel"], md["shard_numel"]
        lay.params = [ParamSpec(p["name"], tuple(p["shape"]), p["numel"], p["full_offset"]) for p in md["params"]]
        lay.groups = [ShardGroup(g["name"], g["full_offset"], g["shard_len"], g["shard_offset"], g["numel"])
                      for g in md["groups"]]
        return lay
