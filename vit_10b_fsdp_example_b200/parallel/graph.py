"""Whole-training-step CUDA graph.

On XLA the reference's Python only *traces* a step and the compiled graph is launched once per iteration
(run_vit_training.py:253 "the first few iterations are very slow due to compilation").  The CUDA
analogue is stream capture: forward, loss, backward (with recompute), the gathers / reduce-scatters on the
communication stream, gradient clipping and the fused AdamW kernels are recorded once and replayed with a single
launch per step.  For launch-bound models (ViT-L and smaller) this removes the ~1000 host launches per step.

Everything that changes from step to step lives in device memory: the batch (static input buffers), the learning
rate and step count (``optimizer.hyper``), the clip coefficient, and the cross-GPU sequence numbers of the
symmetric-memory collectives.
"""
from __future__ import annotations

from typing import Optional

import torch


class GraphedTrainStep:
    """``loss = step(images, target)`` == forward_backward + clip_grad_norm_ + optimizer.step(), graph-replayed.

    The first ``warmup`` calls run eagerly (they also set kernel attributes and fill host-side caches); the next call
    captures; later calls replay.  ``lr_scheduler.step()`` stays on the host: the new learning rate is copied to the
    device before each replay.
    """

    def __init__(self, model, optimizer, clip_grad_norm: float = 0.0, warmup: int = 3):
        cfg = model.cfg
        if model.training and cfg.drop_path_rate > 0:
            raise RuntimeError("CUDA-graph training steps do not support drop_path_rate > 0 "
                               "(masks are keyed from the host)")
        if model.training and cfg.patch_drop_rate > 0:
            raise RuntimeError("CUDA-graph training steps do not support patch_drop_rate > 0 "
                               "(the kept patches are keyed from the host)")
        if model.training and cfg.mixing:
            raise RuntimeError("CUDA-graph training steps do not support mixup / cutmix > 0 "
                               "(lam and the box come from the host)")
        if not model.is_cuda:
            raise RuntimeError("CUDA graphs need a CUDA model")
        if model.training and (cfg.pos_dropout > 0 or cfg.att_dropout > 0 or cfg.mlp_dropout > 0):
            raise RuntimeError("CUDA-graph training steps do not support dropout > 0 (masks are seeded from the host)")
        if getattr(optimizer, "fused", False):
            raise RuntimeError("AdamW fused into the reduce-scatter passes host scalars; use fuse=False with graphs")
        if model.dp_world > 1 and model.backend.name != "sm100":
            raise RuntimeError("multi-GPU CUDA-graph steps need the sm100 (symmetric-memory) backend")
        self.model, self.optimizer = model, optimizer
        self.clip = float(clip_grad_norm)
        self.warmup = warmup
        self.calls = 0
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.images = self.target = self.loss = self.norm = None
        self.launches_per_step = 0  # hand-written kernels recorded in the graph (replays do not pass through Python)

    def _eager(self, images, target):
        loss = self.model.forward_backward(images, target)
        norm = self.model.clip_grad_norm_(self.clip) if self.clip > 0 else None
        self.optimizer.step()
        return loss, norm

    def _capture(self, images, target) -> None:
        model, opt = self.model, self.optimizer
        self.images = images.clone()
        self.target = target.clone()
        opt.lr_on_device = True
        opt.push_lr()
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        n0 = model.ops.launch_count() if hasattr(model.ops, "launch_count") else 0
        with torch.cuda.graph(self.graph):
            self.loss, self.norm = self._eager(self.images, self.target)
        self.launches_per_step = (model.ops.launch_count() - n0) if hasattr(model.ops, "launch_count") else 0
        # capture only records; the host-side step counters advanced once -> undo, replay() advances them again
        for u in model.all_units:
            opt.state[u.name]["step"] -= 1
        model.step_count -= 1

    def __call__(self, images: torch.Tensor, target: torch.Tensor):
        self.calls += 1
        if self.calls <= self.warmup:
            loss, self.norm = self._eager(images, target)
            return loss
        if self.graph is None:
            self._capture(images, target)
        self.images.copy_(images, non_blocking=True)
        self.target.copy_(target, non_blocking=True)
        self.optimizer.push_lr()
        self.graph.replay()
        for u in self.model.all_units:
            self.optimizer.state[u.name]["step"] += 1
        self.model.step_count += 1
        return self.loss

    @property
    def grad_norm(self):
        return self.norm
