"""Sharded AdamW over the FSDP units' flat shards (reference: torch.optim.AdamW over sharded
parameters, run_vit_training.py:237,278-280).

By default the semantics match ``torch.optim.AdamW(lr, weight_decay)`` with default betas (0.9, 0.999) / eps 1e-8 and a
single parameter group: decoupled weight decay is applied to *every* tensor, biases and LayerNorm included
(reference :237).  Because a rank only owns shards, optimizer state is sharded for free (ZeRO).

``filter_bias_and_norm`` / ``layer_decay`` (``--filter_bias_and_norm`` / ``--layer_decay``) switch to MAE / timm
parameter groups (see ``param_groups``): no weight decay on 1-D parameters and the learned tokens, and block i trained at
``lr * layer_decay ** (L - i)``.  The groups reach the kernels as per-unit tables (a group index per 64-element chunk
of the shard and a [G, 2] table of (lr_scale, wd)), so one grouped launch per unit still updates the whole shard.  The
scheduler keeps driving the one base lr, ``param_groups[0]["lr"]``.

One fused kernel per unit reads the reduced gradient shard, applies the clip coefficient armed by
``model.clip_grad_norm_`` (a device scalar: no host sync, no separate scaling pass), updates m / v and the
split-fp32 master, and thereby also produces the bf16 shard the next all-gather ships.  With a model EMA
(``FSDPViT(model_ema=True)``, ``model_ema_decay`` here) the same kernel also updates the EMA from the new master while
it is in registers: ``ema = d * ema + (1 - d) * w`` (timm ModelEmaV2 with a fixed decay).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import param_groups as pg


class ShardedAdamW:
    def __init__(self, model, lr: float = 1e-3, weight_decay: float = 1e-2, betas=(0.9, 0.999), eps: float = 1e-8,
                 fuse_into_reduce_scatter: bool = False, model_ema_decay: Optional[float] = None,
                 filter_bias_and_norm: bool = False, layer_decay: Optional[float] = None):
        """fuse_into_reduce_scatter: apply the update of each unit inside its gradient reduce-scatter kernel while
        backward is still running (sm100 backend, world > 1).  Only legal when gradient clipping is disabled,
        because clipping needs the norm of the whole gradient before any parameter changes.  A model with an EMA
        never takes this route: the reduce-scatter kernel has no EMA operand, so its units are updated by step().

        model_ema_decay: the EMA decay d in [0, 1); required exactly when the model has an EMA.

        filter_bias_and_norm: no weight decay on 1-D parameters, pos_embed, cls_token and reg_token.
        layer_decay: d in (0, 1]: layer-wise lr scales d ** (L + 1 - layer id); implies filter_bias_and_norm."""
        has_ema = bool(getattr(model, "has_ema", False))
        if has_ema and model_ema_decay is None:
            raise ValueError("the model has an EMA: pass model_ema_decay")
        if model_ema_decay is not None:
            if not has_ema:
                raise ValueError("model_ema_decay needs a model with an EMA (FSDPViT(model_ema=True))")
            if not 0.0 <= float(model_ema_decay) < 1.0:
                raise ValueError(f"model_ema_decay must be in [0, 1), got {model_ema_decay}")
        self.ema_decay = float(model_ema_decay) if has_ema else None
        if layer_decay is not None:
            layer_decay = float(layer_decay)
            if not 0.0 < layer_decay <= 1.0:
                raise ValueError(f"layer_decay must be in (0, 1], got {layer_decay}")
            filter_bias_and_norm = True  # as MAE and timm: layer-wise decay comes with the no-decay filter
        self.model = model
        self.param_groups = [dict(lr=lr, weight_decay=weight_decay, betas=tuple(betas), eps=eps,
                                  filter_bias_and_norm=bool(filter_bias_and_norm), layer_decay=layer_decay)]
        # per-unit group tables (static: built before any CUDA-graph capture); None = one group, the plain kernels
        self.groups: Optional[Dict[str, pg.UnitGroups]] = None
        if filter_bias_and_norm:
            self.groups = {u.name: pg.build_unit_groups(model.cfg, u.layout, model.shard_rank, weight_decay, layer_decay,
                                                        model.device) for u in model.all_units}
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
        args = (unit.hi, unit.lo, unit.exp_avg, unit.exp_avg_sq,
                [g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], float(st["step"])])
        if self.groups is None:
            return args
        ug = self.groups[unit.name]
        return args + (ug.chunk_groups, ug.group_hyper)

    def group_summary(self):
        """The parameter groups of the whole model (layer, decay, lr scale, wd, tensors, elements); None without them."""
        return None if self.groups is None else pg.summary(list(self.groups.values()))

    def _group_operands(self, unit) -> dict:
        if self.groups is None:
            return {}
        ug = self.groups[unit.name]
        return {"groups": ug.chunk_groups, "group_hyper": ug.group_hyper}

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
            grp = self._group_operands(u)
            if model.split_master:
                if ema is None:
                    ops.adamw_split(u.hi, u.lo, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd,
                                    st["step"], hyper, **grp)
                else:
                    ops.adamw_split(u.hi, u.lo, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd,
                                    st["step"], hyper, ema=ema, ema_decay=self.ema_decay, **grp)
            elif ema is None:
                ops.adamw_fp32(u.master, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd, st["step"],
                               **grp)
            else:
                ops.adamw_fp32(u.master, u.exp_avg, u.exp_avg_sq, u.shard_grad, clip, lr, b1, b2, eps, wd, st["step"],
                               ema=ema, ema_decay=self.ema_decay, **grp)
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

    def check_group_settings(self, saved: dict) -> None:
        """Refuse optimizer state saved under other parameter-group settings, naming the flag to pass or drop.  State
        without the keys was written before parameter groups existed: both flags off."""
        ld, sld = self.param_groups[0]["layer_decay"], saved.get("layer_decay")
        filt, sfilt = self.param_groups[0]["filter_bias_and_norm"], bool(saved.get("filter_bias_and_norm", False))
        if sld != ld:
            if sld is None:
                raise ValueError(f"the checkpoint was trained without layer-wise lr decay: drop --layer_decay to resume "
                                 f"it{' (keep --filter_bias_and_norm)' if sfilt else ''}")
            raise ValueError(f"the checkpoint was trained with --layer_decay {sld}: pass --layer_decay {sld} to resume it")
        if sfilt != filt:
            if sfilt:
                raise ValueError("the checkpoint was trained with --filter_bias_and_norm (no weight decay on biases, "
                                 "norms and tokens): pass --filter_bias_and_norm to resume it")
            raise ValueError("the checkpoint was trained with weight decay on every tensor: drop --filter_bias_and_norm "
                             "to resume it")

    def load_state_dict(self, sd: dict) -> None:
        self.check_group_settings(sd["param_groups"][0])
        for u in self.model.all_units:
            st = sd["state"][u.name]
            self.state[u.name]["step"] = int(st["step"])
            u.exp_avg.copy_(st["exp_avg"])
            u.exp_avg_sq.copy_(st["exp_avg_sq"])
        if self.hyper is not None and self.model.all_units:
            self.hyper[1] = float(self.state[self.model.all_units[0].name]["step"])
        for g, sg in zip(self.param_groups, sd["param_groups"]):
            g.update({k: (tuple(v) if k == "betas" else v) for k, v in sg.items()
                      if k not in ("filter_bias_and_norm", "layer_decay")})
        if self.groups is not None:  # the decayed rows follow a restored weight_decay (in place: graphs read them)
            wd = float(self.param_groups[0]["weight_decay"])
            for ug in self.groups.values():
                for r in ug.rows:
                    r.weight_decay = wd if r.decay else 0.0
                ug.group_hyper.copy_(torch.tensor([[r.lr_scale, r.weight_decay] for r in ug.rows], dtype=torch.float32))

    def __repr__(self) -> str:
        g = self.param_groups[0]
        return (f"ShardedAdamW(lr={g['lr']}, betas={g['betas']}, eps={g['eps']}, weight_decay={g['weight_decay']}, "
                f"units={len(self.model.all_units)}, clip_fused_into_update={not self.fused}, "
                f"fused_into_reduce_scatter={self.fused}, filter_bias_and_norm={g['filter_bias_and_norm']}, "
                f"layer_decay={g['layer_decay']}"
                f"{'' if self.ema_decay is None else f', model_ema_decay={self.ema_decay}'})")
