"""Hand-rolled fully-sharded data-parallel (ZeRO-3 / ZeRO-2 / DDP) engine for the functional ViT.

What the reference gets from ``XlaFullyShardedDataParallel`` + ``checkpoint_module`` + XLA's scheduler
(run_vit_training.py:165-200, 261-280) is implemented here explicitly:

  * one FSDP unit per transformer block + one root unit (patch/pos embed, final norm, head)   (:145,199)
  * each rank keeps only its shard of every unit's parameters, gradients and AdamW state      (:177-181,237)
  * forward : all-gather unit i+1 (comm stream) while unit i computes; free after use when
              ``reshard_after_forward`` (ZeRO-3) or keep until backward (ZeRO-2-like)            (:174,358)
  * backward: re-gather, recompute the block from its checkpointed input (``grad_ckpt``), run the
              hand-written backward, reduce-scatter (mean) the unit's gradients while the next block
              computes -> 2 all-gathers + 1 reduce-scatter per block per step                    (:194,357)
  * memory-aware extension of ``grad_ckpt``: the top K blocks keep a lean activation set instead of being
              recomputed, K sized from the HBM that is free after the first step (``ckpt_keep_blocks``)
  * ``clip_grad_norm_`` over the *full* gradient (local sum of squares -> all-reduce)           (:266-270)
  * ``--run_without_fsdp``: replicated parameters + gradient all-reduce (DDP comparison mode)   (:171-172,271-275)
  * ``--shard_on_cpu``: blocks are built, sharded on the host one at a time, only shards reach HBM (:175-178)
  * sharded ``state_dict`` / ``load_state_dict`` / ``get_shard_metadata``                       (utils.py:26-40)

Memory layout (bf16 compute): the fp32 master weight of a shard is stored *split* as (bf16 hi, int16 lo);
``hi`` is simultaneously the tensor peers all-gather from, so there is no separate low-precision copy and
no cast pass.  On one GPU the gathered buffer aliases the shard itself (zero-copy).
"""
from __future__ import annotations

import contextlib
import math
import os
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..config import ViTConfig
from ..models import vit
from .backends import make_backend
from .layout import UnitLayout


class _NullEvent:
    def record(self, *a, **k):
        pass

    def wait(self, *a, **k):
        pass

    def synchronize(self):
        pass


# debug aid: overwrite a gathered-parameter buffer with NaN the moment the engine releases it, so any
# use-after-release of resharded parameters shows up as a NaN loss instead of silently reading stale weights
DEBUG_POISON = os.environ.get("B200_DEBUG_POISON", "0") == "1"
# NVTX ranges around every block's forward / backward (visible in nsys / ncu timelines)
NVTX = os.environ.get("B200_NVTX", "0") == "1"

# keep re-materialisable tensors (P, LN outputs, gelu(u)) too when HBM is left over after keeping every block
EXTRAS_ENABLED = os.environ.get("B200_CKPT_EXTRAS", "1") != "0"


class FsdpUnit:
    """Sharded state of one FSDP unit on this rank."""

    def __init__(self, name: str, layout: UnitLayout, index: int):
        self.name, self.layout, self.index = name, layout, index
        self.master: Optional[torch.Tensor] = None   # fp32 shard (fp32 compute mode)
        self.hi: Optional[torch.Tensor] = None       # bf16 shard  (bf16 compute mode; also the all-gather source)
        self.lo: Optional[torch.Tensor] = None       # int16 remainder so (hi<<16)+lo == fp32 master bits
        self.exp_avg: Optional[torch.Tensor] = None
        self.exp_avg_sq: Optional[torch.Tensor] = None
        self.shard_grad: Optional[torch.Tensor] = None
        self.full: Optional[torch.Tensor] = None     # gathered parameters (compute dtype) while resident
        self.full_grad: Optional[torch.Tensor] = None
        self.gather_event = None
        self.reduce_event = None
        self.fused_pending = ()  # weights the next block_forward has to gather itself (AG-fused GEMMs)

    @property
    def compute_shard(self) -> torch.Tensor:
        return self.hi if self.hi is not None else self.master


class FSDPViT:
    """The sharded model: ``loss = model.forward_backward(images, target)``; ``logits = model(images)``."""

    def __init__(self, vcfg: ViTConfig, *, world: int = 1, rank: int = 0, device=None, dtype=torch.float32,
                 reshard_after_forward: bool = True, flatten_parameters: bool = False, grad_ckpt: bool = True,
                 run_without_fsdp: bool = False, shard_on_cpu: bool = False, backend: str = "torchdist",
                 seed: int = 0, init_device: str = "cpu", verbose_build=None, fuse_all_gather: bool = True,
                 ckpt_keep_blocks: int = 0):
        self.cfg = vcfg
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.dtype = dtype
        self.dp_world, self.rank = world, rank
        self.use_fsdp = not run_without_fsdp
        # In DDP comparison mode every rank holds everything: shard math runs with world = 1.
        self.world = world if self.use_fsdp else 1
        self.shard_rank = rank if self.use_fsdp else 0
        self.reshard_after_forward = reshard_after_forward
        self.flatten_parameters = flatten_parameters
        self.grad_ckpt = grad_ckpt
        # Memory-aware activation checkpointing: the top `keep_blocks` blocks keep a lean set of activations
        # (10 [T, D] tensors: nothing a GEMM would have to recompute) and skip the forward recompute in backward;
        # the blocks below are checkpointed as in the reference (run_vit_training.py:171 checkpoint_module).
        # -1 = decide after the first step from the HBM that is actually free (see _auto_keep_blocks).
        self.keep_blocks = int(ckpt_keep_blocks) if grad_ckpt else 0
        # how many of the kept blocks (counted from the top) additionally keep P / both LN outputs / gelu(u)
        # instead of re-materialising them; filled by the automatic policy with whatever HBM is left over
        self.keep_extras = {"P": 0, "h": 0, "g": 0}
        self.shard_on_cpu = shard_on_cpu
        self.training = True
        self.is_cuda = self.device.type == "cuda"
        self.split_master = dtype == torch.bfloat16
        if self.is_cuda:
            from ..ops import cuda_ops

            assert dtype == torch.bfloat16, "the sm_90a kernel path is bf16 (use --device cpu for fp32 reference runs)"
            self.ops = cuda_ops
        else:
            from ..ops import torch_ops

            self.ops = torch_ops
        self.backend = make_backend(backend if self.is_cuda else "torchdist", world, rank, self.device)
        self.drop = vit.DropoutCtx(seed)
        self._clip_coef = None
        self._grad_norm = None
        self._sumsq = None
        self._fused_sumsq = False
        self.step_count = 0        # optimizer steps since the start of training (checkpointed: seeds the dropout masks)
        self._steps_here = 0       # forward_backward calls of THIS process (the keep policy is sized after the first one)
        # All-gather fused into the qkv / fc1 GEMMs (copier warp pulling peer slabs with SM-issued loads): on by default
        # at W = 2 only; with more peers one warp per CTA has to pull (W - 1) / W of the weight while the GEMM waits
        # for it, so the whole block is gathered by the copy engines instead.  The crossover has not been measured on
        # H100 (no multi-GPU run yet).  B200_FUSE_AG=1 / 0 forces either way.
        fuse_env = os.environ.get("B200_FUSE_AG", "")
        self.fuse_all_gather = fuse_all_gather and fuse_env != "0" and (world <= 2 or fuse_env == "1")
        self._stall_probe = None  # list of (event, event) pairs while exposed_comm_probe() is active
        self._unrecorded = set()  # ids of events created but never recorded (must not be waited on during capture)
        self._fused_opt = None  # ShardedAdamW registered for reduce-scatter + AdamW fusion (clipping off only)

        # ---- streams ----
        if self.is_cuda:
            # B200_COMM_PRIORITY=-1 puts the collectives on a high-priority stream (their CTAs are then placed
            # ahead of pending GEMM CTAs instead of at the next kernel tail); default 0 until A/B-measured.
            self.comm_stream = torch.cuda.Stream(device=self.device,
                                                 priority=int(os.environ.get("B200_COMM_PRIORITY", "0")))
        else:
            self.comm_stream = None

        # ---- units: blocks are built / sharded ONE AT A TIME (host peak = one full block) ----
        self.units: List[FsdpUnit] = []
        bspecs, rspecs = vit.block_param_specs(vcfg), vit.root_param_specs(vcfg)
        gen_device = "cpu" if (shard_on_cpu or init_device == "cpu" or not self.is_cuda) else self.device
        for i in range(vcfg.num_blocks):
            lay = UnitLayout.build(f"blocks.{i}", bspecs, self.world, flatten_parameters)
            unit = FsdpUnit(lay.name, lay, i)
            self._init_unit(unit, lambda g, d: vit.init_block_params(vcfg, g, d), seed * 100003 + i + 1, gen_device)
            self.units.append(unit)
            if verbose_build is not None:
                verbose_build(f"built ViT block {i}")  # run_vit_training.py:147
        lay = UnitLayout.build("root", rspecs, self.world, flatten_parameters)
        self.root = FsdpUnit("root", lay, vcfg.num_blocks)
        self._init_unit(self.root, lambda g, d: vit.init_root_params(vcfg, g, d), seed * 100003, gen_device)
        self.blocks = self.units
        self.all_units = self.units + [self.root]

        # ---- transient buffers ----
        self._setup_buffers()
        self.backend.params_updated()

    # ------------------------------------------------------------------------------------------------
    # construction
    # ------------------------------------------------------------------------------------------------
    def _init_unit(self, unit: FsdpUnit, init_fn, seed: int, gen_device) -> None:
        lay = unit.layout
        # Parameters are drawn on the host by default (bit-identical on every rank and in every mode, like the
        # reference which builds each block on CPU); init_device="cuda" draws them with the device Philox
        # generator instead (same values on every rank, ~100x faster for the 10B model).
        gen = torch.Generator(device=gen_device)
        gen.manual_seed(seed)
        params = init_fn(gen, gen_device)  # fp32
        work_dev = "cpu" if (self.shard_on_cpu or not self.is_cuda) else self.device
        full = torch.zeros(lay.full_numel, dtype=torch.float32, device=work_dev)
        for p in lay.params:
            full[p.full_offset: p.full_offset + p.numel].copy_(params[p.name].reshape(-1), non_blocking=False)
        del params
        shard = torch.zeros(lay.shard_numel, dtype=torch.float32, device=work_dev)
        lay.shard_from_full(full, self.shard_rank, shard)
        del full
        self._install_master(unit, shard.to(self.device))
        n = lay.shard_numel
        unit.exp_avg = torch.zeros(n, dtype=torch.float32, device=self.device)
        unit.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=self.device)

    def _install_master(self, unit: FsdpUnit, shard_fp32: torch.Tensor) -> None:
        n = unit.layout.shard_numel
        if self.split_master:
            if unit.hi is None:
                unit.hi = self.backend.alloc_shard(n, torch.bfloat16)
                unit.lo = torch.empty(n, dtype=torch.int16, device=self.device)
            self.ops.split_fp32(shard_fp32, unit.hi, unit.lo)
        else:
            if unit.master is None:
                unit.master = self.backend.alloc_shard(n, torch.float32)
            unit.master.copy_(shard_fp32)

    def master_fp32(self, unit: FsdpUnit) -> torch.Tensor:
        """This rank's fp32 master shard (reconstructed exactly from the split representation)."""
        if not self.split_master:
            return unit.master
        out = torch.empty(unit.layout.shard_numel, dtype=torch.float32, device=self.device)
        self.ops.merge_fp32(unit.hi, unit.lo, out)
        return out

    def _setup_buffers(self) -> None:
        W = self.world
        blocks = self.units
        max_full = max(u.layout.full_numel for u in blocks) if blocks else 0
        self._alias = W == 1  # gathered buffer == shard buffer, gradient buffer == shard gradient
        self._free_events: Dict[int, object] = {}
        if self._alias:
            for u in self.all_units:
                u.full = u.compute_shard
                u.full_grad = self.backend.alloc_full_grad(u.layout.full_numel, self.dtype)
                u.shard_grad = u.full_grad
            self._param_bufs, self._grad_bufs = [], []
            return
        n_param_bufs = 2 if self.reshard_after_forward else len(blocks)
        self._param_bufs = [torch.empty(max_full, dtype=self.dtype, device=self.device) for _ in range(n_param_bufs)]
        self._grad_bufs = [self.backend.alloc_full_grad(max_full, self.dtype) for _ in range(min(2, max(1, len(blocks))))]
        self._param_buf_free = [self._new_event() for _ in self._param_bufs]
        self._grad_buf_free = [self._new_event() for _ in self._grad_bufs]
        self.root.full = torch.empty(self.root.layout.full_numel, dtype=self.dtype, device=self.device)
        self.root.full_grad = self.backend.alloc_full_grad(self.root.layout.full_numel, self.dtype)
        for u in self.all_units:
            u.shard_grad = torch.zeros(u.layout.shard_numel, dtype=torch.float32, device=self.device)
        self._fused_sumsq = self.backend.name == "sm100"

    # ------------------------------------------------------------------------------------------------
    # stream helpers (no-ops on CPU)
    # ------------------------------------------------------------------------------------------------
    @contextlib.contextmanager
    def _range(self, name: str):
        if NVTX and self.is_cuda:
            torch.cuda.nvtx.range_push(name)
            try:
                yield
            finally:
                torch.cuda.nvtx.range_pop()
        else:
            yield

    def _new_event(self):
        return torch.cuda.Event() if self.is_cuda else _NullEvent()

    def _on_comm(self):
        return torch.cuda.stream(self.comm_stream) if self.is_cuda else contextlib.nullcontext()

    def _record(self, ev):
        if self.is_cuda:
            ev.record(torch.cuda.current_stream())
            self._unrecorded.discard(id(ev))
        return ev

    def _wait(self, ev):
        if self.is_cuda and ev is not None and id(ev) not in self._unrecorded:
            cur = torch.cuda.current_stream()
            probe = self._stall_probe is not None and cur != self.comm_stream
            if probe:  # exposed-communication probe: how long the compute stream sits in this wait
                e0 = torch.cuda.Event(enable_timing=True)
                e0.record(cur)
            cur.wait_event(ev)
            if probe:
                e1 = torch.cuda.Event(enable_timing=True)
                e1.record(cur)
                self._stall_probe.append((e0, e1))

    @contextlib.contextmanager
    def exposed_comm_probe(self):
        """``with model.exposed_comm_probe() as r: <steps>`` -> r["ms"] = total time the compute stream spent
        blocked on communication-stream events (all-gather not there yet, reduce-scatter still reading a gradient
        buffer, end-of-step join) and r["waits"] = number of such waits.  This is BASELINE.md's secondary metric
        "exposed comm ms/step".  Event records cost time themselves, so a few tenths of a millisecond per
        ViT-10B step are the measurement floor.  The all-gather slices pulled *inside* the qkv / fc1 GEMMs do not appear here: any
        stall there is part of that GEMM's duration."""
        res = {"ms": 0.0, "waits": 0}
        self._stall_probe = []
        try:
            yield res
        finally:
            pairs, self._stall_probe = self._stall_probe, None
            if self.is_cuda:
                torch.cuda.synchronize(self.device)
                res["ms"] = float(sum(a.elapsed_time(b) for a, b in pairs))
                res["waits"] = len(pairs)

    # ------------------------------------------------------------------------------------------------
    # gather / reduce scheduling
    # ------------------------------------------------------------------------------------------------
    def _param_buf_index(self, unit: FsdpUnit) -> int:
        return unit.index % len(self._param_bufs)

    def _issue_gather(self, unit: FsdpUnit, fuse: bool = False) -> None:
        """Enqueue the unit's all-gather on the comm stream (prefetch).  No-op if already resident.

        fuse=True: the next thing that runs on this unit is a block_forward, so the big weights consumed by
        its qkv / fc1 GEMMs are left out here and pulled by those GEMM kernels themselves (AG fusion)."""
        if self._alias or unit.gather_event is not None:
            return
        exclude = ()
        if fuse and self.fuse_all_gather and unit is not self.root:
            exclude = self.backend.fusable_params(unit.layout)
        if unit is self.root:
            buf = unit.full
            free_ev = None
        else:
            bi = self._param_buf_index(unit)
            buf = self._param_bufs[bi][: unit.layout.full_numel]
            free_ev = self._param_buf_free[bi]
        with self._on_comm():
            self._wait(free_ev)
            self.backend.all_gather(unit.layout, unit.compute_shard, buf, exclude)
            unit.gather_event = self._record(self._new_event())
        unit.full = buf
        unit.fused_pending = exclude

    def _views(self, unit: FsdpUnit):
        """Parameter views of a resident unit; hands pending AG-fusion specs to the first block_forward."""
        p = unit.layout.param_views(unit.full)
        if unit.fused_pending:
            p.ag = {n: self.backend.ag_fuse_spec(unit.layout, unit.compute_shard, unit.full, n)
                    for n in unit.fused_pending}
            unit.fused_pending = ()
        return p

    def _wait_gather(self, unit: FsdpUnit) -> None:
        if not self._alias:
            self._wait(unit.gather_event)

    def _release_params(self, unit: FsdpUnit) -> None:
        """Compute is done with the gathered parameters of this unit (reshard)."""
        if self._alias or unit is self.root:
            return
        if DEBUG_POISON and unit.full is not None:
            unit.full.fill_(float("nan"))
        self._record(self._param_buf_free[self._param_buf_index(unit)])
        unit.full = None
        unit.gather_event = None

    def _grad_views(self, unit: FsdpUnit):
        if self._alias or unit is self.root:
            buf = unit.full_grad
        else:
            gi = unit.index % len(self._grad_bufs)
            self._wait(self._grad_buf_free[gi])  # the reduce-scatter that last read this buffer is done
            buf = self._grad_bufs[gi][: unit.layout.full_numel]
            unit.full_grad = buf
        return unit.layout.param_views(buf)

    def _issue_reduce(self, unit: FsdpUnit) -> None:
        """Gradients of `unit` are complete on the compute stream: reduce-scatter them on the comm stream."""
        if not self.use_fsdp:
            ready = self._record(self._new_event())
            with self._on_comm():
                self._wait(ready)
                self.backend.all_reduce_mean_(unit.full_grad[: unit.layout.full_numel])
                unit.reduce_event = self._record(self._new_event())
            return
        if self._alias:
            return
        ready = self._record(self._new_event())
        adam = self._fused_opt.fused_args(unit) if self._fused_opt is not None else None
        with self._on_comm():
            self._wait(ready)
            if adam is not None:
                self.backend.reduce_scatter(unit.layout, unit.full_grad, unit.shard_grad,
                                            self._sumsq if self._fused_sumsq else None, self.ops, adam=adam)
            else:
                self.backend.reduce_scatter(unit.layout, unit.full_grad, unit.shard_grad,
                                            self._sumsq if self._fused_sumsq else None, self.ops)
            ev = self._record(self._new_event())
        unit.reduce_event = ev
        if unit is not self.root:
            self._grad_buf_free[unit.index % len(self._grad_bufs)] = ev

    # ------------------------------------------------------------------------------------------------
    # training step: forward + backward
    # ------------------------------------------------------------------------------------------------
    def train(self):
        self.training = True
        self.drop.training = True
        return self

    def eval(self):
        self.training = False
        self.drop.training = False
        return self

    def _begin_step(self) -> None:
        """Fork the communication stream from the compute stream (training step AND inference pass).  Everything the
        previous step / pass enqueued has been joined back into the compute stream -- reductions are waited for at the
        end of forward_backward, buffer releases are recorded on the compute stream itself, the optimizer step and
        its cross-GPU barrier run there, a replayed CUDA graph is ordered on it -- so after this fork every older
        buffer-free event is implied and is replaced by a fresh, not-yet-recorded one.  That also keeps events recorded
        inside a graph capture from ever being waited on by eager code (and vice versa), which CUDA rejects."""
        if not self.is_cuda or self._alias:
            return
        self._param_buf_free = [self._new_event() for _ in self._param_bufs]
        self._grad_buf_free = [self._new_event() for _ in self._grad_bufs]
        self._unrecorded = set(id(e) for e in self._param_buf_free + self._grad_buf_free)
        for u in self.all_units:  # a gather left over from an earlier pass is stale: the shards may have changed
            u.gather_event = None
        fork = self._record(self._new_event())
        with self._on_comm():
            self._wait(fork)

    def lean_bytes_per_block(self, batch: int) -> int:
        """HBM a block's lean activation set occupies: x, qkv (3), attention out, x1, fc1 pre-activation.  With QK
        normalisation the set keeps the un-normalised qkv plus the norm's fp32 mean and rstd per (token, q or k, head):
        16 bytes per token and head (16.8 MB per ViT-10B block at 128 images, against about 3.4 GB for the rest).
        Every image has cfg.train_tokens rows in a training step (prefix tokens included, dropped patches not)."""
        cfg = self.cfg
        T = cfg.train_tokens
        units = 6.0 + cfg.mlp_ratio
        n = int(batch * T * cfg.embed_dim * units * torch.empty((), dtype=self.dtype).element_size())
        if cfg.qk_norm:
            n += 16 * batch * T * cfg.num_heads
        return n

    def _auto_keep_blocks(self, batch: int) -> int:
        """Called once, after the first (fully checkpointed) step: the caching allocator now holds that step's
        transient peak, so whatever the device still reports free can hold kept activations.  The margin covers
        allocator fragmentation; the result is the minimum over ranks so every GPU runs the same schedule."""
        if not self.is_cuda:
            return 0
        if self.dp_world > 1:
            dist.all_reduce(torch.zeros(1, device=self.device))  # communicator buffers exist before we measure
        torch.cuda.synchronize(self.device)
        free, total = torch.cuda.mem_get_info(self.device)
        margin = int(float(os.environ.get("B200_CKPT_MARGIN_GB", "8")) * 2 ** 30) + total // 50
        k = max(0, min(len(self.units), (free - margin) // max(1, self.lean_bytes_per_block(batch))))
        # left-over HBM: keep re-materialisable tensors too, best saving per byte first (P, LN outputs, gelu(u))
        # (only 60 % of it: the extras change the allocation pattern, keep slack for allocator fragmentation)
        left = int(0.6 * (free - margin - k * self.lean_bytes_per_block(batch)))
        extras = []
        for name, nbytes in self.extra_bytes_per_block(batch):
            if nbytes <= 0:  # nothing to keep for this slot (P under the fused attention pair)
                extras.append(0)
                continue
            n = int(max(0, min(k, left // nbytes))) if k == len(self.units) and EXTRAS_ENABLED else 0
            left -= n * nbytes
            extras.append(n)
        vals = [k] + extras
        if self.dp_world > 1:
            t = torch.tensor(vals, dtype=torch.int64, device=self.device)
            dist.all_reduce(t, op=dist.ReduceOp.MIN)
            vals = [int(v) for v in t.tolist()]
        self.keep_extras = dict(zip(("P", "h", "g"), vals[1:]))
        return int(vals[0])

    def extra_bytes_per_block(self, batch: int):
        cfg = self.cfg
        es = torch.empty((), dtype=self.dtype).element_size()
        T = cfg.train_tokens  # tokens per image in a training step
        unit = batch * T * cfg.embed_dim * es
        npad = (T + 7) // 8 * 8
        # with the fused attention pair (forward keeps the row log-sum-exp, backward rebuilds P tile by tile) there is
        # no P to keep: its budget goes to the LayerNorm outputs and gelu(u) instead
        flash = bool(getattr(self.ops, "use_flash", lambda n, hd: False)(T, cfg.head_dim))
        p_bytes = 0 if flash else batch * cfg.num_heads * T * npad * es
        # g is [T, mlp_out_dim]: mlp_ratio units, or mlp_ratio / 2 with SwiGLU (the lean set's u is [T, Hd] either way)
        return (("P", p_bytes), ("h", 2 * unit), ("g", int(cfg.mlp_out_dim / cfg.embed_dim * unit)))

    def _save_mode(self, i: int, keep_from: int):
        """What block i stores in forward: False = only its input (checkpoint), True = everything
        (--no_grad_ckpt), else the set of extras kept on top of the lean set."""
        if not self.grad_ckpt:
            return True
        if i < keep_from:
            return False
        top = len(self.units) - 1 - i  # 0 for the top block: its activations are released first in backward
        return frozenset(n for n, cnt in self.keep_extras.items() if top < cnt)

    def forward_backward(self, images: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """One micro-step: loss, and this rank's (mean-reduced) shard gradients in ``unit.shard_grad``."""
        cfg, ops = self.cfg, self.ops
        B = images.shape[0]
        blocks = self.units
        if self.keep_blocks < 0:
            # (not step_count: a resumed run starts with step_count > 0 but has not seen its transient peak yet)
            if self._steps_here == 0 or (self.is_cuda and torch.cuda.is_current_stream_capturing()):
                n_keep = 0
            else:
                self.keep_blocks = n_keep = self._auto_keep_blocks(B)
        else:
            n_keep = min(self.keep_blocks, len(blocks))
        keep_from = len(blocks) - n_keep if self.grad_ckpt else 0  # blocks >= keep_from are not recomputed
        self.drop.step = self.step_count
        # global index of this rank's first image (every rank holds the same local batch): stochastic depth draws its
        # per-sample masks there, in FSDP and in --run_without_fsdp mode alike
        self.drop.sample_offset = self.rank * B
        # Mixup / CutMix: one host draw per step, keyed by (seed, step_count, rank); this rank mixes image b with image
        # B-1-b of its own local batch inside the im2col, and the loss takes the matching soft targets
        mix = None
        if cfg.mixing:
            if B % 2:
                raise ValueError(f"--mixup / --cutmix pair image b with image B-1-b and need an even local batch, "
                                 f"got {B}")
            mix = vit.draw_mix(cfg, vit.mix_rng(self.drop.seed, self.step_count, self.rank))
        loss_kw = {}
        if mix is not None:
            loss_kw["mix"] = mix
        if cfg.smoothing > 0:
            loss_kw["smoothing"] = cfg.smoothing
        self._begin_step()
        if self._fused_sumsq:
            self._sumsq = torch.zeros(1, dtype=torch.float32, device=self.device)
        # -------- forward --------
        self._issue_gather(self.root)
        if blocks:
            self._issue_gather(blocks[0], fuse=True)
        self._wait_gather(self.root)
        rp = self.root.layout.param_views(self.root.full)
        x, stem_saved = vit.stem_forward(ops, cfg, rp, images, self.dtype, self.drop, mix=mix)
        ckpt: List[torch.Tensor] = []
        saved_all = []
        for i, u in enumerate(blocks):
            if i + 1 < len(blocks):
                self._issue_gather(blocks[i + 1], fuse=True)
            self._wait_gather(u)
            p = self._views(u)
            with self._range(f"fwd block {i}"):
                if i < keep_from:
                    ckpt.append(x)
                    x, _ = vit.block_forward(ops, cfg, p, x, B, save=False, drop=self.drop, block_idx=i)
                else:
                    x, s = vit.block_forward(ops, cfg, p, x, B, save=self._save_mode(i, keep_from), drop=self.drop,
                                             block_idx=i)
                    saved_all.append(s)
            if self.reshard_after_forward and i != len(blocks) - 1:
                self._release_params(u)  # the last block is needed again immediately by backward
        logits, head_saved = vit.head_forward(ops, cfg, rp, x, B)
        loss, dlogits, _ = ops.cross_entropy(logits, target, want_grad=True, **loss_kw)
        # -------- backward --------
        rg = self._grad_views(self.root)
        dx, dx_sum = vit.head_backward(ops, cfg, rp, rg, head_saved, dlogits, B)
        del head_saved, logits, dlogits
        for i in range(len(blocks) - 1, -1, -1):
            u = blocks[i]
            # a recomputed block runs its qkv / fc1 forward GEMMs again and those pull their own weights
            self._issue_gather(u, fuse=i < keep_from)
            if i - 1 >= 0:
                self._issue_gather(blocks[i - 1], fuse=i - 1 < keep_from)  # prefetch for the backward sweep
            self._wait_gather(u)
            p = self._views(u)
            with self._range(f"bwd block {i}"):
                if i < keep_from:
                    xin = ckpt.pop()
                    _, s = vit.block_forward(ops, cfg, p, xin, B, save=True, drop=self.drop, block_idx=i)
                else:
                    s = saved_all.pop()
                g = self._grad_views(u)
                dx, dx_sum = vit.block_backward(ops, cfg, p, g, s, dx, dx_sum, B)
                del s
            self._release_params(u)
            self._issue_reduce(u)
        vit.stem_backward(ops, cfg, rp, rg, stem_saved, dx, dx_sum)
        self._issue_reduce(self.root)
        self.root.gather_event = None  # parameters change in the optimizer step: re-gather next step
        # compute stream must not run ahead of the reductions it depends on (optimizer / clip read them)
        for u in self.all_units:
            self._wait(u.reduce_event)
            u.reduce_event = None
        self.step_count += 1
        self._steps_here += 1
        return loss

    # ------------------------------------------------------------------------------------------------
    # inference
    # ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        cfg, ops = self.cfg, self.ops
        B = images.shape[0]
        blocks = self.units
        self._begin_step()  # the gathers below must not overtake the optimizer step / barrier on the compute stream
        self._issue_gather(self.root)
        if blocks:
            self._issue_gather(blocks[0], fuse=True)
        self._wait_gather(self.root)
        rp = self.root.layout.param_views(self.root.full)
        drop = self.drop if self.training else None
        self.drop.sample_offset = self.rank * B
        x, _ = vit.stem_forward(ops, cfg, rp, images, self.dtype, drop)
        for i, u in enumerate(blocks):
            if i + 1 < len(blocks):
                self._issue_gather(blocks[i + 1], fuse=True)
            self._wait_gather(u)
            x, _ = vit.block_forward(ops, cfg, self._views(u), x, B, save=False, drop=drop, block_idx=i)
            self._release_params(u)
        logits, _ = vit.head_forward(ops, cfg, rp, x, B)
        self.root.gather_event = None
        return logits

    # ------------------------------------------------------------------------------------------------
    # gradient clipping (norm of the FULL gradient) -- reference :266-270
    # ------------------------------------------------------------------------------------------------
    def clip_grad_norm_(self, max_norm: float) -> torch.Tensor:
        """Computes the global gradient norm and arms the clip coefficient consumed by the next
        ``optimizer.step()`` (the scaling is fused into the AdamW kernel instead of a separate pass)."""
        ops = self.ops
        if self._fused_opt is not None:
            raise RuntimeError("clip_grad_norm_ cannot be used with AdamW fused into the reduce-scatter: the update "
                               "has already been applied during backward (construct the optimizer with fuse=False)")
        if self._fused_sumsq and self._sumsq is not None:
            total = self._sumsq
        else:
            total = torch.zeros(1, dtype=torch.float32, device=self.device)
            for u in self.all_units:
                ops.sumsq(u.shard_grad, total)
        if self.use_fsdp:
            self.backend.all_reduce_scalars_(total, "sum")
        coef, norm = ops.clip_coef(total, float(max_norm))
        self._clip_coef, self._grad_norm = coef, norm
        return norm

    # ------------------------------------------------------------------------------------------------
    # parameters / state
    # ------------------------------------------------------------------------------------------------
    def parameters(self) -> List[torch.Tensor]:
        """The tensors this rank owns (shards only, like FSDP's ``model.parameters()``; reference :233)."""
        return [u.compute_shard for u in self.all_units]

    def num_sharded_parameters(self) -> int:
        return sum(u.layout.shard_numel for u in self.all_units)

    def num_parameters(self) -> int:
        return sum(u.layout.payload_numel() for u in self.all_units)

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Only this rank's shards (fp32, on host), keyed ``<unit>.<param>`` or ``<unit>.flat_param``."""
        out = {}
        for u in self.all_units:
            m = self.master_fp32(u).detach().cpu()
            for g in u.layout.groups:
                out[f"{u.name}.{g.name}"] = m[g.shard_offset: g.shard_offset + g.shard_len].clone()
        return out

    def load_state_dict(self, state: Dict[str, torch.Tensor], shard_metadata: Optional[dict] = None) -> None:
        if shard_metadata and "step_count" in shard_metadata:
            self.step_count = int(shard_metadata["step_count"])
        for u in self.all_units:
            m = torch.empty(u.layout.shard_numel, dtype=torch.float32)
            for g in u.layout.groups:
                t = state[f"{u.name}.{g.name}"]
                assert t.numel() == g.shard_len, f"shard size mismatch for {u.name}.{g.name} (world size changed?)"
                m[g.shard_offset: g.shard_offset + g.shard_len].copy_(t)
            self._install_master(u, m.to(self.device))
        self.backend.params_updated()

    def load_full_state_dict(self, full: Dict[str, torch.Tensor]) -> None:
        """Initialise this rank's shards from a *consolidated* (unsharded, timm-style) state_dict, e.g. the output
        of ``consolidate_sharded_ckpts``: the way to continue a run on a different number of GPUs, which per-rank
        shard files alone cannot do (``load_state_dict`` asserts the world size is unchanged)."""
        has_qk = any(k.endswith(("attn.q_norm.weight", "attn.k_norm.weight")) for k in full)
        if self.cfg.qk_norm and not has_qk:
            raise ValueError("this model uses --qk_norm, but the checkpoint has no attn.q_norm / attn.k_norm "
                             "parameters: it was trained without QK normalisation")
        if has_qk and not self.cfg.qk_norm:
            raise ValueError("the checkpoint has attn.q_norm / attn.k_norm parameters (it was trained with QK "
                             "normalisation): pass --qk_norm to load it")
        has_ls = any(k.endswith(("ls1.gamma", "ls2.gamma")) for k in full)
        if self.cfg.init_values and not has_ls:
            raise ValueError("this model uses --init_values (LayerScale), but the checkpoint has no ls1.gamma / "
                             "ls2.gamma parameters: it was trained without LayerScale")
        if has_ls and not self.cfg.init_values:
            raise ValueError("the checkpoint has ls1.gamma / ls2.gamma parameters (it was trained with LayerScale): "
                             "pass --init_values to load it (any value > 0; the learned gammas are loaded)")
        self.check_prefix_tokens(full)
        self.check_mlp_form(full)
        for u in self.all_units:
            lay = u.layout
            prefix = "" if u is self.root else u.name + "."
            buf = torch.zeros(lay.full_numel, dtype=torch.float32)
            for p in lay.params:
                t = full[prefix + p.name].detach().to(torch.float32).cpu()
                if p.name == "patch_embed.proj.weight":  # [D, 3, P, P] -> [D, 3*P*P] zero-padded to the TMA-legal K
                    t = t.reshape(p.shape[0], -1)
                    t = torch.nn.functional.pad(t, (0, p.shape[1] - t.shape[1]))
                assert t.numel() == p.numel, f"{prefix + p.name}: {tuple(t.shape)} does not match {p.shape}"
                buf[p.full_offset: p.full_offset + p.numel].copy_(t.reshape(-1))
            shard = torch.zeros(lay.shard_numel, dtype=torch.float32)
            lay.shard_from_full(buf, self.shard_rank, shard)
            self._install_master(u, shard.to(self.device))
        self.backend.params_updated()

    def check_mlp_form(self, full: Dict[str, torch.Tensor]) -> None:
        """Refuse a consolidated checkpoint whose MLP form does not match --swiglu, read from the shapes: an fc2 input
        width equal to half the fc1 rows is SwiGLU (timm SwiGLUPacked), an equal width is the GELU MLP."""
        key = next((k for k in full if k.endswith("mlp.fc1.weight")), None)
        if key is None or key[: -len("fc1.weight")] + "fc2.weight" not in full:
            return
        rows, width = full[key].shape[0], full[key[: -len("fc1.weight")] + "fc2.weight"].shape[-1]
        glu = 2 * width == rows
        if self.cfg.swiglu and not glu:
            raise ValueError(f"this model uses --swiglu, but the checkpoint's MLP is not SwiGLU ({key} has {rows} rows "
                             f"and fc2 reads {width} features, not {rows // 2}): drop --swiglu to load it")
        if glu and not self.cfg.swiglu:
            raise ValueError(f"the checkpoint's MLP is SwiGLU ({key} has {rows} rows and fc2 reads half of them, "
                             f"{width}): pass --swiglu to load it")

    def check_prefix_tokens(self, full: Dict[str, torch.Tensor]) -> None:
        """Refuse a consolidated checkpoint whose prefix-token layout (class token, register tokens, rows of pos_embed)
        does not match this model's flags, naming the flag to pass or drop.  pos_embed may hold another grid (the
        caller resamples it); what must match is whether its first P rows belong to the prefix tokens."""
        cfg, D = self.cfg, self.cfg.embed_dim
        has_cls = "cls_token" in full
        if cfg.class_token and not has_cls:
            raise ValueError("this model uses --class_token, but the checkpoint has no cls_token: it was trained "
                             "without a class token (drop --class_token to load it)")
        if has_cls and not cfg.class_token:
            raise ValueError("the checkpoint has a cls_token (it was trained with a class token): pass --class_token "
                             "to load it")
        n_reg = full["reg_token"].numel() // D if "reg_token" in full else 0
        if n_reg != cfg.reg_tokens:
            fix = f"pass --reg_tokens {n_reg}" if n_reg else "drop --reg_tokens"
            raise ValueError(f"the checkpoint has {n_reg} register tokens (reg_token) and this model "
                             f"{cfg.reg_tokens}: {fix} to load it")
        if not cfg.class_token or "pos_embed" not in full:
            return
        rows = full["pos_embed"].numel() // D

        def grid_fits(n: int) -> bool:
            return n >= 1 and math.isqrt(n) ** 2 == n

        P = cfg.num_prefix_tokens
        if grid_fits(rows - (0 if cfg.no_embed_class else P)):
            return
        if cfg.no_embed_class and grid_fits(rows - P):
            raise ValueError(f"the checkpoint's pos_embed has {rows} rows, {P} prefix tokens plus a square grid: the "
                             f"prefix tokens were position-embedded, drop --no_embed_class to load it")
        if cfg.class_token and not cfg.no_embed_class and grid_fits(rows):
            raise ValueError(f"the checkpoint's pos_embed has {rows} rows, a square grid without the {P} prefix "
                             f"tokens: pass --no_embed_class to load it")
        want = "a square grid" if cfg.no_embed_class else f"{P} prefix rows plus a square grid"
        raise ValueError(f"the checkpoint's pos_embed has {rows} rows, but this model needs {want}")

    def get_shard_metadata(self) -> dict:
        """Everything the offline consolidation tool needs to rebuild full tensors (reference utils.py:29)."""
        return {
            "world_size": self.world, "rank": self.shard_rank, "flatten_parameters": self.flatten_parameters,
            "fsdp": self.use_fsdp, "units": [u.layout.metadata() for u in self.all_units],
            "step_count": int(self.step_count),  # seeds the dropout masks: a resumed run must not replay epoch 1's
            "logical_shapes": {k: list(v) for k, v in vit.logical_shapes(self.cfg).items()},
            "patch_k": self.cfg.patch_k,
            "model": {k: getattr(self.cfg, k) for k in ("image_size", "patch_size", "embed_dim", "num_heads",
                                                        "num_blocks", "mlp_ratio", "num_classes", "class_token",
                                                        "reg_tokens", "no_embed_class", "swiglu")},
        }

    def __repr__(self) -> str:
        c = self.cfg
        mode = "FSDP(ZeRO-3)" if self.use_fsdp and self.reshard_after_forward else (
            "FSDP(ZeRO-2)" if self.use_fsdp else "DDP")
        return (f"FSDPViT[{mode}, world={self.dp_world}, backend={self.backend.name}, ops={self.ops.NAME}, "
                f"dtype={self.dtype}]("
                f"image={c.image_size}, patch={c.patch_size}, dim={c.embed_dim}, heads={c.num_heads}, "
                f"blocks={c.num_blocks}, mlp_ratio={c.mlp_ratio}, classes={c.num_classes}, "
                f"grad_ckpt={self.grad_ckpt}, flatten={self.flatten_parameters}, "
                f"params={self.num_parameters():,}, sharded={self.num_sharded_parameters():,})")
