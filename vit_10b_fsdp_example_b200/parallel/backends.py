"""Collective backends of the FSDP engine.

``TorchDistBackend``  torch.distributed collectives (gloo on CPU, NCCL on GPU).  It is the CPU test vehicle
                      and the honest NCCL baseline -- *not* the product path on H100.
``Sm100Backend``      hand-written NVLink / NVSwitch kernels over symmetric memory (csrc/comm.cu):
                      sync-free peer-to-peer all-gather that lands shards in their final position,
                      one-pass reduce-scatter (+1/W mean, +fp32 cast, +grad-norm partial) with optional
                      in-switch NVLS reduction, flag barriers and scalar all-reduce.  No NCCL on the hot path.

Both implement the same small interface used by ``engine.FSDPViT``:
    alloc_shard / alloc_full_grad / all_gather / reduce_scatter / all_reduce_scalars_ / all_reduce_mean_ / barrier
(replaces torch_xla's XLA collectives + xm.mesh_reduce / xm.rendezvous, reference run_vit_training.py:177-181,
205,224,270,273).
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist

from .layout import UnitLayout


class TorchDistBackend:
    name = "torchdist"
    supports_fused_adam = False

    def __init__(self, world: int, rank: int, device: torch.device):
        self.world, self.rank, self.device = world, rank, device
        self.is_gloo = world > 1 and dist.get_backend() == "gloo"
        self._staging = {}

    # ---- allocation (plain device memory) ----
    def alloc_shard(self, numel: int, dtype) -> torch.Tensor:
        return torch.zeros(numel, dtype=dtype, device=self.device)

    def alloc_full_grad(self, numel: int, dtype) -> torch.Tensor:
        return torch.zeros(numel, dtype=dtype, device=self.device)

    # ---- collectives ----
    def fusable_params(self, layout: UnitLayout):
        return ()

    def all_gather(self, layout: UnitLayout, shard: torch.Tensor, out_full: torch.Tensor, exclude=()) -> None:
        if self.world == 1:
            if out_full.data_ptr() != shard.data_ptr():
                out_full[: shard.numel()].copy_(shard)
            return
        if len(layout.groups) == 1:  # flat parameter: the gathered tensor *is* the full buffer
            dist.all_gather_into_tensor(out_full[: layout.full_numel], shard)
            return
        staging = torch.empty(self.world * layout.shard_numel, dtype=shard.dtype, device=shard.device)
        dist.all_gather_into_tensor(staging, shard)
        st = staging.view(self.world, layout.shard_numel)
        for g in layout.groups:  # copy-out (this pass is what the P2P kernel avoids)
            out_full[g.full_offset: g.full_offset + self.world * g.shard_len].view(self.world, g.shard_len).copy_(
                st[:, g.shard_offset: g.shard_offset + g.shard_len])

    def reduce_scatter(self, layout: UnitLayout, full_grad: torch.Tensor, out_shard: torch.Tensor,
                       sumsq: Optional[torch.Tensor] = None, ops=None) -> None:
        """out_shard (fp32) = mean over ranks of this rank's slices of full_grad; sumsq += |out_shard|^2."""
        W = self.world
        if W == 1:
            if out_shard.data_ptr() != full_grad.data_ptr():
                out_shard.copy_(full_grad[: out_shard.numel()])
        else:
            # one fp32 staging buffer per shard size, reused across calls (collectives on one stream are serialised, so
            # the previous user is done): the NCCL / gloo backend is the honest baseline, not a handicapped one
            key = (layout.shard_numel, str(full_grad.device))
            staging = self._staging.get(key)
            if staging is None:
                staging = self._staging[key] = torch.empty(W, layout.shard_numel, dtype=torch.float32,
                                                           device=full_grad.device)
            for g in layout.groups:  # copy-in, fp32 so the reduction accumulates in fp32
                staging[:, g.shard_offset: g.shard_offset + g.shard_len].copy_(
                    full_grad[g.full_offset: g.full_offset + W * g.shard_len].view(W, g.shard_len))
            if self.is_gloo:
                dist.all_reduce(staging)
                out_shard.copy_(staging[self.rank])
            else:
                dist.reduce_scatter_tensor(out_shard, staging.view(-1))
            out_shard.mul_(1.0 / W)
        if sumsq is not None:
            ops.sumsq(out_shard, sumsq)

    def all_reduce_scalars_(self, t: torch.Tensor, op: str = "sum") -> torch.Tensor:
        if self.world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM if op == "sum" else dist.ReduceOp.MAX)
        return t

    def all_reduce_mean_(self, t: torch.Tensor) -> torch.Tensor:
        """DDP-style gradient all-reduce (reference --run_without_fsdp, xm.reduce_gradients :273)."""
        if self.world > 1:
            if t.dtype == torch.bfloat16 and self.is_gloo:
                f = t.float()
                dist.all_reduce(f)
                t.copy_(f.mul_(1.0 / self.world))
            else:
                dist.all_reduce(t)
                t.mul_(1.0 / self.world)
        return t

    def barrier(self) -> None:
        if self.world > 1:
            dist.barrier()

    def step_begin(self) -> None:
        pass

    def params_updated(self) -> None:
        pass


class Sm100Backend(TorchDistBackend):
    """Symmetric-memory NVLink backend.  Falls back to the parent (NCCL) only for host-side utilities."""

    name = "sm100"
    FLAG_BYTES = 64 * 1024  # flags: uint32[slot][16]; scratch floats follow at +32 KiB

    # flag slots in the symmetric control region (uint32 [slot][16]): 0 params_updated barrier, 1-2 stand-alone
    # barriers (tests), 4-5 scalar all-reduce, 6-7 "inputs ready" / "done reading" of reduce-scatter & all-reduce
    SLOT_READY, SLOT_DONE, RS_COUNTER = 6, 7, 5

    def __init__(self, world: int, rank: int, device: torch.device, comm_ctas: int = 64):
        super().__init__(world, rank, device)
        from ..ops import native

        self._C = native.load()
        # Collective kernels are light CTAs (128 threads, <= 96 registers, no shared memory, see csrc/comm.cu);
        # comm_ctas bounds how many of them one collective launches.  The value has not been tuned on H100.
        self.comm_ctas = int(os.environ.get("B200_COMM_CTAS", comm_ctas))
        # stand-alone all-gather transport: "kernel" = light pull kernel (csrc/comm.cu), "ce" = copy engines.
        # The copy engines take nothing from the SMs, so they are the default; the two transports have not been
        # compared on H100.
        self.ag_transport = os.environ.get("B200_AG_TRANSPORT", "ce")
        self.use_nvls = False
        if world == 1:  # single GPU: nothing to communicate, gathered buffers alias the shards
            return
        import torch.distributed._symmetric_memory as symm_mem

        self._symm = symm_mem
        self._handles = []   # keep rendezvous handles alive
        self._peer = {}      # data_ptr of a symmetric tensor -> list of peer base pointers
        self._mc = {}        # data_ptr -> multicast base pointer (0 if unsupported)
        self._seg_cache = {}
        # per-slot sequence numbers live on the device (advanced inside the kernels), so every collective launch is
        # replayable from a CUDA graph; all ranks issue the same sequence of collectives, hence identical counters
        self._seq_dev = torch.zeros(16, dtype=torch.int32, device=device)
        self._cta_ctr = torch.zeros(1, dtype=torch.int32, device=device)  # last-CTA detection inside the collectives
        self.group_name = dist.group.WORLD.group_name
        ctrl = self._symm_alloc(self.FLAG_BYTES, torch.uint8)
        ctrl.zero_()
        self._ctrl = ctrl
        self._flag_ptrs = self._peer[ctrl.data_ptr()]
        self._scratch_ptrs = [p + 32 * 1024 for p in self._flag_ptrs]
        torch.cuda.synchronize()
        dist.barrier()
        self.use_nvls = all(v != 0 for v in self._mc.values()) and os.environ.get("B200_NVLS", "1") != "0"
        # timing experiment only (wrong numerics): every "peer" pointer is this rank's own buffer and the barriers
        # are skipped -> same kernels, same HBM traffic and SM footprint, but no NVLink traffic and no cross-rank waits
        self._local_only = os.environ.get("B200_COMM_LOCAL", "0") == "1"
        if self._local_only:
            self.use_nvls = False

    # ---- symmetric allocation ----
    def _symm_alloc(self, numel: int, dtype) -> torch.Tensor:
        t = self._symm.empty(numel, dtype=dtype, device=self.device)
        hdl = self._symm.rendezvous(t, dist.group.WORLD)
        self._handles.append((t, hdl))
        self._peer[t.data_ptr()] = [int(p) for p in hdl.buffer_ptrs]
        if os.environ.get("B200_COMM_LOCAL", "0") == "1":
            self._peer[t.data_ptr()] = [int(t.data_ptr())] * self.world
        mc = 0
        try:
            if hdl.has_multicast_support:
                mc = int(hdl.multicast_ptr)
        except Exception:
            mc = 0
        self._mc[t.data_ptr()] = mc
        return t

    def alloc_shard(self, numel: int, dtype) -> torch.Tensor:
        if self.world == 1:
            return super().alloc_shard(numel, dtype)
        t = self._symm_alloc(numel, dtype)
        t.zero_()
        return t

    def alloc_full_grad(self, numel: int, dtype) -> torch.Tensor:
        if self.world == 1:
            return super().alloc_full_grad(numel, dtype)
        t = self._symm_alloc(numel, dtype)
        t.zero_()
        return t

    def device_barrier(self, slot: int = 0) -> None:
        """Stream-ordered cross-GPU barrier on the current stream (flags in symmetric memory)."""
        if getattr(self, "_local_only", False):
            return
        self._C.signal_barrier(self._flag_ptrs, self.rank, self.world, slot, 0, self._seq_dev)

    # ---- segment tables (device int64), built once per (layout, purpose) ----
    @staticmethod
    def _lay_key(layout: UnitLayout):
        """Structural identity of a layout (id() of a short-lived layout object can be recycled by the allocator)."""
        return (layout.name, layout.world, layout.flatten, layout.full_numel,
                tuple((g.name, g.full_offset, g.shard_len, g.shard_offset) for g in layout.groups))

    def _ag_table(self, layout: UnitLayout, esize: int, exclude=()):
        """Segment table of the pull all-gather.  The order of the rows is the order in which this rank's CTAs walk
        the sources, so it is staggered by rank and rotated every MiB: at any moment the W ranks pull from W
        *different* peers.  (With every rank walking the sources 0, 1, 2 ... in the same order all of them would hit
        one GPU's egress at once.)"""
        key = ("ag", self._lay_key(layout), esize, tuple(sorted(exclude)))
        if key not in self._seg_cache:
            chunk = self._C.ag_chunk_bytes()
            piece = 64 * chunk  # 1 MiB per (source, turn)
            rows, prefix = [], 0
            W = self.world
            for g in layout.groups:
                if g.name in exclude:
                    continue  # gathered by the GEMM that consumes it (AG fusion)
                nbytes = g.shard_len * esize
                for pi, off in enumerate(range(0, nbytes, piece)):
                    n = min(piece, nbytes - off)
                    for k in range(W):
                        r = (self.rank + k + pi) % W
                        rows.append([r, g.shard_offset * esize + off, (g.full_offset + r * g.shard_len) * esize + off,
                                     n, prefix])
                        prefix += -(-n // chunk)
            self._seg_cache[key] = (torch.tensor(rows, dtype=torch.int64, device=self.device), prefix)
        return self._seg_cache[key]

    # ---- all-gather fused into the consuming GEMM ----
    FUSED_PARAMS = ("attn.qkv.weight", "mlp.fc1.weight")

    def fusable_params(self, layout: UnitLayout):
        """Weights whose all-gather can run inside the forward GEMM that consumes them: per-parameter shard
        groups made of whole rows (dim-0 slabs), no padding.  A SwiGLU fc1 (fc2 reads half its rows) is left to the
        unit all-gather: its GEMM tiles read a gate and a value row range, which sit in two different slabs."""
        if self.world == 1 or layout.flatten:
            return ()
        shapes = {p.name: p.shape for p in layout.params}
        glu = ("mlp.fc1.weight" in shapes and "mlp.fc2.weight" in shapes
               and 2 * shapes["mlp.fc2.weight"][1] == shapes["mlp.fc1.weight"][0])
        ok = []
        for g in layout.groups:
            if g.name not in self.FUSED_PARAMS or (glu and g.name == "mlp.fc1.weight"):
                continue
            spec = next(p for p in layout.params if p.name == g.name)
            rows, cols = spec.shape
            if rows % self.world == 0 and g.shard_len == (rows // self.world) * cols and (g.shard_len * 2) % 16 == 0:
                ok.append(g.name)
        return tuple(ok)

    def ag_fuse_spec(self, layout: UnitLayout, shard: torch.Tensor, full_buf: torch.Tensor, name: str):
        """Argument list for `_C.gemm(..., ag=...)`: the kernel pulls every rank's slab of `name` itself."""
        g = next(x for x in layout.groups if x.name == name)
        spec = next(p for p in layout.params if p.name == name)
        esize = shard.element_size()
        key = ("flags", full_buf.data_ptr(), name)
        if key not in self._seg_cache:
            # one arrival counter per slab, then the chunk counter of the copier warps at [world] (gemm_sm90.cu zeroes
            # world + 1 words before every launch)
            self._seg_cache[key] = torch.zeros(self.world + 1, dtype=torch.int32, device=self.device)
        flags = self._seg_cache[key]
        peers = [p + g.shard_offset * esize for p in self._peer[shard.data_ptr()]]
        return [self.world, self.rank, spec.shape[0] // self.world, g.shard_len * esize,
                full_buf.data_ptr() + g.full_offset * esize, flags.data_ptr()] + peers

    def _rs_table(self, layout: UnitLayout, esize: int):
        key = ("rs", self._lay_key(layout), esize)
        if key not in self._seg_cache:
            chunk = self._C.rs_chunk_vecs() * (16 // esize)  # elements per chunk (one CTA pass of 16-byte vectors)
            rows, prefix = [], 0
            for (foff, soff, n) in layout.scatter_segments(self.rank):
                rows.append([foff * esize, soff, n, prefix])
                prefix += -(-n // chunk)
            self._seg_cache[key] = (torch.tensor(rows, dtype=torch.int64, device=self.device), prefix)
        return self._seg_cache[key]

    # ---- collectives ----
    def all_gather(self, layout: UnitLayout, shard: torch.Tensor, out_full: torch.Tensor, exclude=()) -> None:
        if self.world == 1:
            return super().all_gather(layout, shard, out_full)
        # (inside a CUDA-graph capture the pull kernel is used: it is the transport the graphed multi-GPU step was
        # validated with; memcpy nodes between peer-mapped allocations are untested there)
        if self.ag_transport == "ce" and not torch.cuda.is_current_stream_capturing():
            src, dst, nb = self._ag_copies(layout, shard, out_full, exclude)
            self._C.ce_all_gather(src, dst, nb)
            return
        table, chunks = self._ag_table(layout, shard.element_size(), exclude)
        self._C.p2p_all_gather(self._peer[shard.data_ptr()], self.rank, out_full, table, chunks, self.comm_ctas)

    def _ag_copies(self, layout: UnitLayout, shard: torch.Tensor, out_full: torch.Tensor, exclude=()):
        """(src, dst, nbytes) lists of the copy-engine all-gather: one copy per (group, source rank), sources walked
        starting at this rank's successor so the W ranks read from W different peers at any time."""
        key = ("agce", self._lay_key(layout), shard.data_ptr(), out_full.data_ptr(), tuple(sorted(exclude)))
        if key not in self._seg_cache:
            es = shard.element_size()
            peers = self._peer[shard.data_ptr()]
            src, dst, nb = [], [], []
            for k in range(self.world):
                r = (self.rank + 1 + k) % self.world  # own slice last: it is the only copy that does not need NVLink
                for g in layout.groups:
                    if g.name in exclude:
                        continue
                    src.append(peers[r] + g.shard_offset * es)
                    dst.append(out_full.data_ptr() + (g.full_offset + r * g.shard_len) * es)
                    nb.append(g.shard_len * es)
            self._seg_cache[key] = (src, dst, nb)
        return self._seg_cache[key]

    supports_fused_adam = True

    def reduce_scatter(self, layout: UnitLayout, full_grad: torch.Tensor, out_shard: torch.Tensor,
                       sumsq: Optional[torch.Tensor] = None, ops=None, adam=None) -> None:
        """adam = (hi, lo, m, v, [lr, beta1, beta2, eps, wd, step]) fuses the sharded AdamW update into the kernel
        (legal only without gradient clipping); out_shard is then left untouched."""
        if self.world == 1:
            return super().reduce_scatter(layout, full_grad, out_shard, sumsq, ops)
        table, chunks = self._rs_table(layout, full_grad.element_size())
        scale = 1.0 / self.world
        a = tuple(adam) if adam is not None else (None, None, None, None, [])
        bf16 = full_grad.dtype == torch.bfloat16
        mc = self._mc[full_grad.data_ptr()] if (self.use_nvls and bf16) else 0
        # ONE kernel: publish "gradients complete" -> wait for the peers' -> reduce -> publish "done reading" ->
        # wait until every peer is done (after which the gradient buffer may be overwritten)
        self._C.reduce_scatter(self._peer[full_grad.data_ptr()], mc, self.rank, self.world, out_shard, table, chunks,
                               bf16, scale, sumsq, self.comm_ctas, *self._sync_args(), *a)

    def _sync_args(self):
        if self._local_only:  # timing experiment: no cross-rank flags
            return [], [], None, None
        return ([self.rank, self.world, self.SLOT_READY, self.SLOT_DONE, self.RS_COUNTER], self._flag_ptrs,
                self._seq_dev, self._cta_ctr)

    def all_reduce_mean_(self, t: torch.Tensor) -> torch.Tensor:
        """DDP gradient all-reduce (--run_without_fsdp; reference xm.reduce_gradients, run_vit_training.py:273) on the
        symmetric gradient buffer: in-switch multimem.ld_reduce + multimem.st (or pull-reduce-push over peer
        pointers), same in-kernel flag protocol as the reduce-scatter.  No NCCL."""
        if self.world == 1:
            return t
        ptr = t.data_ptr()
        if ptr not in self._peer or t.dtype != torch.bfloat16 or (t.numel() * 2) % 16 != 0 or self._local_only:
            return super().all_reduce_mean_(t)  # not a symmetric gradient buffer: NCCL utility path
        mc = self._mc[ptr] if self.use_nvls else 0
        self._C.all_reduce_mean(self._peer[ptr], mc, self.rank, self.world, t, self.comm_ctas, *self._sync_args())
        return t

    def all_reduce_scalars_(self, t: torch.Tensor, op: str = "sum") -> torch.Tensor:
        if self.world > 1 and not self._local_only:
            assert t.dtype == torch.float32 and t.numel() <= 16
            # flag / scratch slot 4 or 5, alternating with the device-side sequence number (counter 3)
            self._C.allreduce_scalars(self._flag_ptrs, self._scratch_ptrs, self.rank, self.world, 4, 0, t,
                                      0 if op == "sum" else 1, self._seq_dev, 3)
        return t

    def params_updated(self) -> None:
        """Shards were rewritten by the optimizer: peers may only pull them after everyone is done."""
        if self.world > 1:
            self.device_barrier(slot=0)


def make_backend(kind: str, world: int, rank: int, device: torch.device):
    if kind == "sm100":
        return Sm100Backend(world, rank, device)
    return TorchDistBackend(world, rank, device)
