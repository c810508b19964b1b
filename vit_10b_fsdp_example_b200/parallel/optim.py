"""Sharded AdamW over the FSDP units' flat shards (reference: torch.optim.AdamW over sharded
parameters, run_vit_training.py:237,278-280).

Semantics match ``torch.optim.AdamW(lr, weight_decay)`` with default betas (0.9, 0.999) / eps 1e-8 and a
single parameter group: decoupled weight decay is applied to *every* tensor, biases and LayerNorm included
(reference :237).  Because a rank only owns shards, optimizer state is sharded for free (ZeRO).

One fused kernel per unit reads the reduced gradient shard, applies the clip coefficient armed by
``model.clip_grad_norm_`` (a device scalar: no host sync, no separate scaling pass), updates m / v and the
split-fp32 master, and thereby also produces the bf16 shard the next all-gather ships.  With a model EMA
(``FSDPViT(model_ema=True)``, ``model_ema_decay`` here) the same kernel also updates the EMA from the new master while
it is in registers: ``ema = d * ema + (1 - d) * w`` (timm ModelEmaV2 with a fixed decay).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch


class ShardedAdamW:
    def __init__(self, model, lr: float = 1e-3, weight_decay: float = 1e-2, betas=(0.9, 0.999), eps: float = 1e-8,
                 fuse_into_reduce_scatter: bool = False, model_ema_decay: Optional[float] = None):
        """fuse_into_reduce_scatter: apply the update of each unit inside its gradient reduce-scatter kernel while
        backward is still running (sm100 backend, world > 1).  Only legal when gradient clipping is disabled,
        because clipping needs the norm of the whole gradient before any parameter changes.  A model with an EMA
        never takes this route: the reduce-scatter kernel has no EMA operand, so its units are updated by step().

        model_ema_decay: the EMA decay d in [0, 1); required exactly when the model has an EMA."""
        has_ema = bool(getattr(model, "has_ema", False))
        if has_ema and model_ema_decay is None:
            raise ValueError("the model has an EMA: pass model_ema_decay")
        if model_ema_decay is not None:
            if not has_ema:
                raise ValueError("model_ema_decay needs a model with an EMA (FSDPViT(model_ema=True))")
            if not 0.0 <= float(model_ema_decay) < 1.0:
                raise ValueError(f"model_ema_decay must be in [0, 1), got {model_ema_decay}")
        self.ema_decay = float(model_ema_decay) if has_ema else None
        self.model = model
        self.param_groups = [dict(lr=lr, weight_decay=weight_decay, betas=tuple(betas), eps=eps)]
        self.state: Dict[str, dict] = {u.name: {"step": 0} for u in model.all_units}
        self.fused = bool(fuse_into_reduce_scatter and model.use_fsdp and model.world > 1 and model.split_master
                          and getattr(model.backend, "supports_fused_adam", False) and not has_ema)
        self._done_in_backward = set()
        if self.fused:
            model._fused_opt = self
        # device-resident [lr, step]: lets the AdamW launches be replayed from a CUDA graph (see parallel/graph.py)
        self.hyper = None
        if model.is_cuda and model.split_master:
            self.hyper = torch.zeros(2, dtype=torch.float32, device=model.device)
        self.lr_on_device = False  # True while a CUDA-graph owner keeps hyper[0] up to date itself

    def push_lr(self) -> None:
        """Write the current host learning rate into the device hyper-parameter block.  The value travels as a
        kernel argument of the fill, so every queued step sees exactly the learning rate it was enqueued with (a
        pinned staging scalar would be re-read by copies that have not executed yet when the host runs ahead)."""
        self.hyper[0:1].fill_(float(self.param_groups[0]["lr"]))

    def fused_args(self, unit):
        """Called by the engine when it enqueues the reduce-scatter of `unit` (fused mode)."""
        g = self.param_groups[0]
        st = self.state[unit.name]
        st["step"] += 1
        self._done_in_backward.add(unit.name)
        return (unit.hi, unit.lo, unit.exp_avg, unit.exp_avg_sq,
                [g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], float(st["step"])])

    def step(self) -> None:
        model, ops = self.model, self.model.ops
        g = self.param_groups[0]
        lr, wd, (b1, b2), eps = g["lr"], g["weight_decay"], g["betas"], g["eps"]
        clip = model._clip_coef
        hyper = self.hyper if not self._done_in_backward else None
        if hyper is not None:
            if not self.lr_on_device:
                self.push_lr()
            hyper[1:2].add_(1.0)  # device-side step counter (all units share the step count)
        for u in model.all_units:
            if u.name in self._done_in_backward:
                continue  # already updated inside its reduce-scatter kernel
            st = self.state[u.name]
            st["step"] += 1
            ema = model.ema_operand(u) if self.ema_decay is not None else None
            if model.split_master:
                if ema is None:
                    ops.adamw_split(u.hi, u.lo, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd,
                                    st["step"], hyper)
                else:
                    ops.adamw_split(u.hi, u.lo, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd,
                                    st["step"], hyper, ema=ema, ema_decay=self.ema_decay)
            elif ema is None:
                ops.adamw_fp32(u.master, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd, st["step"])
            else:
                ops.adamw_fp32(u.master, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd, st["step"],
                               ema=ema, ema_decay=self.ema_decay)
        self._done_in_backward.clear()
        model._clip_coef = None
        model.backend.params_updated()

    def zero_grad(self, set_to_none: bool = True) -> None:
        """Gradient buffers are preallocated and fully overwritten by the next backward / reduce-scatter,
        so there is nothing to free or memset (reference :280 frees grads to save memory)."""
        self.model._clip_coef = None

    def state_dict(self) -> dict:
        state = {}
        for u in self.model.all_units:
            state[u.name] = {"step": self.state[u.name]["step"], "exp_avg": u.exp_avg.detach().cpu().clone(),
                             "exp_avg_sq": u.exp_avg_sq.detach().cpu().clone()}
        groups = [{k: v for k, v in g.items()} for g in self.param_groups]
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd: dict) -> None:
        for u in self.model.all_units:
            st = sd["state"][u.name]
            self.state[u.name]["step"] = int(st["step"])
            u.exp_avg.copy_(st["exp_avg"])
            u.exp_avg_sq.copy_(st["exp_avg_sq"])
        if self.hyper is not None and self.model.all_units:
            self.hyper[1] = float(self.state[self.model.all_units[0].name]["step"])
        for g, sg in zip(self.param_groups, sd["param_groups"]):
            g.update({k: (tuple(v) if k == "betas" else v) for k, v in sg.items()})

    def __repr__(self) -> str:
        g = self.param_groups[0]
        return (f"ShardedAdamW(lr={g['lr']}, betas={g['betas']}, eps={g['eps']}, weight_decay={g['weight_decay']}, "
                f"units={len(self.model.all_units)}, clip_fused_into_update={not self.fused}, "
                f"fused_into_reduce_scatter={self.fused}"
                f"{'' if self.ema_decay is None else f', model_ema_decay={self.ema_decay}'})")
