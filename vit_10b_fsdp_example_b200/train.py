"""Training driver on the H100-native engine.

Capability parity with the reference's driver (run_vit_training.py:203-324): datasets -> sharded model -> AdamW +
warmup-cosine schedule -> optional resume -> epochs of [step, log every ``log_step_interval`` steps] -> per-rank
sharded checkpoint every ``ckpt_epoch_interval`` epochs -> top-1 evaluation every ``test_epoch_interval`` epochs.
The *log line* (``epoch E step S, lr: ..., loss: ..., sec/iter: ..., GPU memory: ...``) and the checkpoint file names
are kept because downstream tooling parses them; the structure is this engine's own:

  ``TrainStep``     one optimisation step (forward + loss + hand-written backward with overlapped collectives, clip on
                    the norm of the FULL gradient, sharded AdamW) -- eager, or replayed as ONE CUDA graph; both are the
                    same callable, so the loop below has a single body.
  ``DeviceClock``   ms/step measured on the device with CUDA events, max over ranks (wall-clock time of an
                    asynchronously launched step measures the host, not the GPU).
  ``Trainer``       owns the pieces and the epoch loop.
"""
from __future__ import annotations

import json
import os
import pprint
import time
from typing import Optional

import torch

from .config import ViTConfig
from .data import build_datasets
from .launch import Runtime
from .parallel import FSDPViT, GraphedTrainStep, ShardedAdamW
from .utils import SmoothedValue, get_warmup_cosine_scheduler
from .utils.checkpoint import load_ckpt, normalize_full_state_dict_keys, resize_pos_embed, save_ckpt


def resolve_dtype(cfg, device: torch.device) -> torch.dtype:
    if cfg.dtype == "auto":
        return torch.bfloat16 if device.type == "cuda" else torch.float32
    return torch.bfloat16 if cfg.dtype == "bf16" else torch.float32


def spans_multiple_hosts() -> bool:
    """True when a torchrun job has more ranks than this host has processes (the reference's pod launch,
    README.md:99-101).  The symmetric-memory kernels need every peer on the same NVSwitch domain."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_WORLD_SIZE", str(world)))
    return world > local


def resolve_backend(cfg, device: torch.device) -> str:
    if cfg.backend == "auto":
        if device.type != "cuda":
            return "torchdist"
        # one NVSwitch box: hand-written P2P / NVLS kernels; several hosts: NCCL collectives (torch.distributed)
        return "torchdist" if spans_multiple_hosts() else "sm100"
    if cfg.backend == "sm100" and spans_multiple_hosts():
        raise ValueError("--backend sm100 needs all ranks on one NVLink/NVSwitch box; use --backend nccl across hosts")
    return "sm100" if cfg.backend == "sm100" else "torchdist"


def resolve_init_device(cfg, device: torch.device) -> str:
    """Where the random initial parameters are drawn.  ``--shard_on_cpu`` is the reference's host-offload path
    (run_vit_training.py:175-178): blocks are built and sharded on the host one at a time.  Otherwise a CUDA run draws
    them with the device generator (same values on every rank, ~100x faster for 10 B parameters) -- the path bench.py
    times; ``--init_device cpu`` keeps host-side generation (bit-identical to a CPU run)."""
    want = getattr(cfg, "init_device", "auto")
    if cfg.shard_on_cpu or device.type != "cuda":
        return "cpu"
    return "cuda" if want in ("auto", "cuda") else "cpu"


def build_fsdp_vit_model(cfg, rt: Runtime) -> FSDPViT:
    """Per-block FSDP units + a root unit, activation checkpointing, optional host-side sharding
    (what reference build_fsdp_vit_model does at run_vit_training.py:165-200)."""
    keep = getattr(cfg, "ckpt_keep_blocks", 0)
    return FSDPViT(
        ViTConfig.from_args(cfg), world=rt.world, rank=rt.rank, device=rt.device, dtype=resolve_dtype(cfg, rt.device),
        reshard_after_forward=cfg.reshard_after_forward, flatten_parameters=cfg.flatten_parameters,
        grad_ckpt=cfg.grad_ckpt, run_without_fsdp=cfg.run_without_fsdp, shard_on_cpu=cfg.shard_on_cpu,
        backend=resolve_backend(cfg, rt.device), seed=cfg.seed, verbose_build=rt.master_print,
        init_device=resolve_init_device(cfg, rt.device),
        ckpt_keep_blocks=keep if rt.device.type == "cuda" else max(0, keep),
        model_ema=bool(getattr(cfg, "model_ema", False)),
    )


class TrainStep:
    """``loss = step(images, target)``: forward, loss, backward, clip, parameter update.

    In FSDP mode the gradients leave ``forward_backward`` already reduce-scattered (mean) and the clip coefficient is
    computed from the norm of the full gradient (reference :266-270); in ``--run_without_fsdp`` mode they were
    all-reduced inside ``forward_backward`` (reference :273) and the same clip applies to the replicated gradient.
    Without clipping the AdamW update is fused into each unit's reduce-scatter kernel (sm100 backend), except with a
    model EMA: that is updated by the stand-alone AdamW kernel, so every unit takes that route.
    """

    def __init__(self, model: FSDPViT, cfg, device: torch.device):
        self.model = model
        self.clip = float(cfg.clip_grad_norm)
        want_graph = bool(getattr(cfg, "cuda_graph", False)) and device.type == "cuda"
        self.optimizer = ShardedAdamW(model, lr=cfg.lr, weight_decay=cfg.weight_decay,
                                      fuse_into_reduce_scatter=self.clip <= 0 and not want_graph and not model.has_ema,
                                      model_ema_decay=float(cfg.model_ema_decay) if model.has_ema else None)
        self.graph: Optional[GraphedTrainStep] = (
            GraphedTrainStep(model, self.optimizer, self.clip) if want_graph else None)

    def __call__(self, images: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        if self.graph is not None:
            return self.graph(images, target)
        loss = self.model.forward_backward(images, target)
        if self.clip > 0:
            self.model.clip_grad_norm_(self.clip)
        self.optimizer.step()
        return loss


class DeviceClock:
    """Device time per step between two ``lap()`` calls: CUDA events, max over ranks; host time on CPU."""

    def __init__(self, rt: Runtime):
        self.rt = rt
        self.cuda = rt.device.type == "cuda"
        self._mark()

    def _mark(self):
        if self.cuda:
            self.ev = torch.cuda.Event(enable_timing=True)
            self.ev.record()
        else:
            self.t = time.time()

    def lap(self, steps: int) -> float:
        if self.cuda:
            prev, _ = self.ev, self._mark()
            self.ev.synchronize()
            ms = prev.elapsed_time(self.ev) / max(1, steps)
        else:
            prev, _ = self.t, self._mark()
            ms = (self.t - prev) * 1e3 / max(1, steps)
        return self.rt.mesh_reduce("step_ms", ms, max)


def format_log_line(epoch: int, step: int, lr: float, loss: float, sec_per_iter: float, images_per_sec: float,
                    memory: dict) -> str:
    """The reference's step line (run_vit_training.py:207-213) with device-timed images/sec added."""
    return (f"epoch {epoch} step {step}, lr: {lr:.4f}, loss: {loss:.4f}, sec/iter: {sec_per_iter:.4f}, "
            f"images/sec: {images_per_sec:.1f}, GPU memory: {memory}")


@torch.no_grad()
def evaluate(rt: Runtime, loader, model: FSDPViT, max_steps: int = 0):
    """Top-1 accuracy over the validation loader; counts are summed over ranks (reference :303-318)."""
    model.eval()
    hits = torch.zeros(1, dtype=torch.long, device=rt.device)
    seen = 0
    for i, (images, target) in enumerate(loader):
        hits += (model(images).argmax(dim=-1) == target.view(-1)).sum()
        seen += target.numel()
        if max_steps and i + 1 >= max_steps:
            break
    correct = rt.mesh_reduce("local_correct", int(hits.item()), sum)
    total = rt.mesh_reduce("local_total", seen, sum)
    return correct / max(total, 1), correct, total


eval_on_val = evaluate  # reference name (run_vit_training.py:303)


def fault_injection_point(rank: int, epoch: int, step: int) -> None:
    """``B200_INJECT_FAILURE=<rank>:<epoch>:<step>`` makes that rank die there without any clean-up (as a crashed
    process would).  Used by the tests of the failure contract: the launcher tears the job down with a non-zero exit
    code instead of leaving the survivors hanging in a collective, and ``--resume_epoch`` continues from the last
    checkpoint (the reference's contract: README.md:100, run_vit_training.py:246-248)."""
    spec = os.environ.get("B200_INJECT_FAILURE")
    if spec and spec == f"{rank}:{epoch}:{step}":
        print(f"[fault injection] rank {rank} dies at epoch {epoch} step {step}", flush=True)
        os._exit(13)


class Trainer:
    def __init__(self, rt: Runtime, cfg):
        self.rt, self.cfg = rt, cfg
        say = rt.master_print
        if ViTConfig.from_args(cfg).mixing and (cfg.batch_size // rt.world) % 2:
            raise ValueError(f"--mixup / --cutmix mix image b with image B-1-b of each rank's batch and need an even "
                             f"local batch; --batch_size {cfg.batch_size} over {rt.world} ranks gives "
                             f"{cfg.batch_size // rt.world}")
        (self.train_set, self.train_loader, self.train_sampler,
         _, self.val_loader, _) = build_datasets(cfg, rt.device, rt.world, rt.rank, log=say)
        rt.rendezvous("loaded dataset")
        say(f"\n=== dataset ===\n{pprint.pformat(self.train_set)}\n")

        self.model = build_fsdp_vit_model(cfg, rt)
        rt.rendezvous("loaded model")
        say(f"\n=== model ===\n{pprint.pformat(self.model)}\n")
        say(f"per-GPU (sharded) parameter num: {sum(p.numel() for p in self.model.parameters())}")

        self.step_fn = TrainStep(self.model, cfg, rt.device)
        self.optimizer = self.step_fn.optimizer
        self.lr_scheduler = get_warmup_cosine_scheduler(
            self.optimizer, warmup_iteration=cfg.warmup_steps,
            max_iteration=len(self.train_set) // cfg.batch_size * cfg.num_epochs)
        rt.rendezvous("loaded optimizer")
        say(f"\n=== optimizer ===\n{pprint.pformat(self.optimizer)}\n")

        if getattr(cfg, "init_from_full_ckpt", ""):
            full = torch.load(cfg.init_from_full_ckpt, map_location="cpu", weights_only=False)
            self.model.load_full_state_dict(self._full_state(full.get("model", full)))
            say(f"parameters initialised from the consolidated checkpoint {cfg.init_from_full_ckpt}")
            if self.model.has_ema:
                if isinstance(full.get("model_ema"), dict):
                    self.model.load_full_state_dict(self._full_state(full["model_ema"]), ema=True)
                    say("model EMA initialised from the checkpoint's model_ema")
                else:
                    say("the checkpoint has no model_ema: the model EMA starts from the loaded weights")
            del full
        os.makedirs(cfg.ckpt_dir, exist_ok=True)
        if cfg.resume_epoch > 0:  # every rank restores its own shard file
            load_ckpt(self._ckpt_path(cfg.resume_epoch), self.model, self.optimizer, self.lr_scheduler)
        self.loss_meter = SmoothedValue(window_size=5)
        self.time_meter = SmoothedValue(window_size=5)

    def _full_state(self, state: dict) -> dict:
        """A consolidated state_dict made ready for load_full_state_dict: wrapper prefixes stripped, the prefix-token
        layout checked, pos_embed resampled to this model's grid."""
        say, mcfg = self.rt.master_print, self.model.cfg
        state = normalize_full_state_dict_keys(state)
        self.model.check_prefix_tokens(state)  # before resampling: a wrong prefix layout is named, not resampled
        if "pos_embed" in state:
            pos = state["pos_embed"]
            P = 0 if mcfg.no_embed_class else mcfg.num_prefix_tokens  # rows of pos_embed that are not the grid
            state["pos_embed"] = resize_pos_embed(pos, mcfg.num_patches, mcfg.embed_dim, num_prefix_tokens=P)
            if state["pos_embed"] is not pos:
                say(f"pos_embed resampled from {pos.shape[1] - P} to {mcfg.num_patches} tokens (bicubic)")
        return state

    def _ckpt_path(self, epoch: int) -> str:
        # One file per *global* rank.  The reference keys the files by the host-local ordinal (:220,247,298), which is
        # the same thing on one host but makes the hosts of a pod overwrite each other on a shared file system and
        # leaves the consolidation tool without ranks >= 8; the global rank is identical on one box and right on many.
        return os.path.join(self.cfg.ckpt_dir, f"epoch_{epoch}_rank_{self.rt.rank}.ckpt")

    # ---- logging: runs as a step closure, i.e. after the step's device work has been enqueued ----
    def _log(self, epoch: int, step: int, loss: torch.Tensor, lr: float, step_ms: float) -> None:
        rt, cfg = self.rt, self.cfg
        self.loss_meter.update(rt.mesh_reduce("loss_value", loss.item(), sum) / rt.world, batch_size=1)
        ips = cfg.batch_size / (step_ms * 1e-3) if step_ms and step_ms > 0 else float("nan")
        rt.master_print(format_log_line(epoch, step + 1, lr, self.loss_meter.avg, self.time_meter.avg, ips,
                                        rt.get_memory_info()))
        if cfg.bench_json and rt.rank == 0:
            with open(cfg.bench_json, "a") as f:
                f.write(json.dumps({"epoch": epoch, "step": step + 1, "lr": lr, "loss": self.loss_meter.avg,
                                    "sec_per_iter": self.time_meter.avg, "images_per_sec": ips}) + "\n")

    def run_epoch(self, epoch: int, first_epoch: bool) -> None:
        rt, cfg = self.rt, self.cfg
        self.model.train()
        self.train_sampler.set_epoch(epoch)
        clock = DeviceClock(rt)
        host_t = time.time()
        since_log = 0
        for step, (images, target) in enumerate(self.train_loader):
            fault_injection_point(rt.rank, epoch, step + 1)
            loss = self.step_fn(images, target)
            self.lr_scheduler.step()
            self.optimizer.zero_grad(set_to_none=True)
            now = time.time()
            self.time_meter.update(now - host_t, batch_size=1)
            host_t = now
            since_log += 1
            if (first_epoch and step == 0) or (step + 1) % cfg.log_step_interval == 0:
                step_ms = clock.lap(since_log)
                since_log = 0
                rt.add_step_closure(self._log, args=(epoch, step, loss, self.optimizer.param_groups[0]["lr"], step_ms))
            rt.run_step_closures()
            if cfg.max_steps and step + 1 >= cfg.max_steps:
                break

    def fit(self):
        rt, cfg = self.rt, self.cfg
        rt.rendezvous("training begins")
        rt.master_print("training begins (kernels are precompiled: no warm-up compilation)")
        for epoch in range(cfg.resume_epoch + 1, cfg.num_epochs + 1):
            rt.master_print(f"starting epoch {epoch}")
            t0 = time.time()
            self.run_epoch(epoch, first_epoch=epoch == cfg.resume_epoch + 1)
            rt.master_print(f"epoch {epoch} done ({time.time() - t0:.2f} sec)")
            last = epoch == cfg.num_epochs
            if epoch % cfg.ckpt_epoch_interval == 0 or last:  # every rank writes its own shards
                save_ckpt(self._ckpt_path(epoch), self.model, self.optimizer, self.lr_scheduler, master_only=False,
                          rank=rt.rank, barrier=rt.rendezvous)
            if epoch % cfg.test_epoch_interval == 0 or last:
                accuracy, _, _ = evaluate(rt, self.val_loader, self.model, max_steps=cfg.max_steps)
                rt.master_print(f"accuracy on val: {accuracy:.4f}")
                if self.model.has_ema:
                    with self.model.ema_weights():
                        accuracy, _, _ = evaluate(rt, self.val_loader, self.model, max_steps=cfg.max_steps)
                    rt.master_print(f"accuracy of the EMA on val: {accuracy:.4f}")
        return self.model, self.optimizer, self.lr_scheduler


def train(rt: Runtime, cfg):
    return Trainer(rt, cfg).fit()


def main(rt: Runtime, cfg):
    if rt.device.type == "cuda":
        # the activation-keeping policy sizes itself from free HBM; segments that can grow avoid fragmentation
        # (the allocator reads this when the first CUDA tensor is created, which has not happened yet)
        os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
    rt.master_print(f"\n=== cfg ===\n{pprint.pformat(cfg)}\n")
    train(rt, cfg)
    rt.master_print("training completed")
