"""Vision Transformer as an explicit functional graph with hand-written forward *and* backward.

Architecture parity with the reference model (run_vit_training.py:99-162, timm 0.4.12 blocks):
  * PatchEmbed = Conv2d(3, D, k=s=P) -> tokens; learned pos_embed; dropout           (:124-129,156-157)
  * num_blocks pre-LN blocks: x += proj(attn(norm1(x))); x += fc2(gelu(fc1(norm2(x))))  (:133-141)
    - optional SwiGLU MLP (timm SwiGLUPacked = GluMlp(act_layer=SiLU, gate_last=False), off in the reference):
      u = fc1(norm2(x)) of width Hd = [gate | value], x += fc2(silu(u[:, :Hd/2]) * u[:, Hd/2:]); the gate runs in the
      fc1 GEMM epilogue and its gradient in the fc2 dgrad epilogue, as GELU's do
    - LayerNorm eps 1e-5 inside blocks, qkv_bias=True, exact (erf) GELU
    - optional QK normalisation (timm Attention(qk_norm=True), off in the reference): q and k of every head go through
      LayerNorm(head_dim, eps 1e-5) (attn.q_norm / attn.k_norm, one weight and bias shared by the heads) before q k^T
    - optional stochastic depth (timm drop_path, off in the reference): x += drop_path(branch) for both branches,
      one Bernoulli per sample and branch, kept samples scaled by 1 / keep_prob, block i at rate
      linspace(0, drop_path_rate, num_blocks)[i], nothing dropped in eval
    - optional LayerScale (CaiT, timm VisionTransformer(init_values=...), off in the reference):
      x += ls1.gamma * branch and x += ls2.gamma * branch, learned per-channel [D] vectors that start at init_values, in
      training and in eval.  The scale is folded into the branch's last layer, gamma o (a W^T + b) = a (gamma o W)^T +
      gamma o b, so the GEMMs run unchanged on the folded weight; the backward recovers dW, db and dgamma from the wgrad
      of the un-scaled weight in one pass over the weight (ops.layer_scale_bwd)
  * optional Mixup / CutMix (timm Mixup, mode 'batch', off in the reference): drawn on the host per step (draw_mix),
    applied inside the patch im2col, with the mixed, smoothed target handled by the cross-entropy
  * optional prefix tokens (timm VisionTransformer(class_token=True, reg_tokens=R), off in the reference): a learned
    cls_token and R reg_tokens in front of every image's N patch tokens, T = N + P tokens with P = 1 + R; pos_embed
    covers all T tokens, or only the patches with no_embed_class.  The patch GEMM still adds the patch rows of pos_embed
    in its epilogue; ops.tokens_fwd / tokens_bwd assemble and split the [B*T, D] token buffer
  * optional patch dropout (timm PatchDropout(prob=R, num_prefix_tokens=P, ordered=True), off in the reference): in
    training every image keeps K = max(1, int(N * (1 - R))) of its patches, drawn on the GPU (ops.patch_drop_select);
    only they go through the im2col and the patch GEMM, with their own pos_embed rows, and every block runs on
    T' = P + K tokens.  Evaluation keeps all patches
  * final LayerNorm(eps=1e-6), mean-pool over tokens (no CLS token), Linear head      (:151-153,159-161);
    with a class token: LayerNorm of the B class rows only (it acts per row) and the head on them
Parameter names are timm-compatible (``norm1.weight``, ``attn.qkv.weight``, ``mlp.fc1.bias`` ...).

There is no autograd here: every stage has an explicit backward, which is what lets the FSDP engine
place every gather / reduce-scatter / free deterministically and write weight gradients straight into
the flat per-unit gradient buffer.  ``ops`` is either ``torch_ops`` (reference, CPU) or ``cuda_ops``
(sm_90a kernels); both expose the same functions.
"""
from __future__ import annotations

import functools
import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from ..config import ViTConfig

BLOCK_LN_EPS = 1e-5  # timm Block default norm_layer=nn.LayerNorm (eps 1e-5)
FINAL_LN_EPS = 1e-6  # run_vit_training.py:151


# ------------------------------------------------------------------------------------------------
# Parameter inventory
# ------------------------------------------------------------------------------------------------
def block_param_specs(cfg: ViTConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    D, Hd, hd, Ho = cfg.embed_dim, cfg.hidden_dim, cfg.head_dim, cfg.mlp_out_dim
    qk = [("attn.q_norm.weight", (hd,)), ("attn.q_norm.bias", (hd,)),
          ("attn.k_norm.weight", (hd,)), ("attn.k_norm.bias", (hd,))] if cfg.qk_norm else []
    ls = [("ls1.gamma", (D,)), ("ls2.gamma", (D,))] if cfg.init_values else []
    return [
        ("norm1.weight", (D,)), ("norm1.bias", (D,)),
        ("attn.qkv.weight", (3 * D, D)), ("attn.qkv.bias", (3 * D,)),
        *qk,  # timm's state_dict order
        ("attn.proj.weight", (D, D)), ("attn.proj.bias", (D,)),
        *ls[:1],  # timm's Block registers ls1 / ls2 after attn / mlp
        ("norm2.weight", (D,)), ("norm2.bias", (D,)),
        ("mlp.fc1.weight", (Hd, D)), ("mlp.fc1.bias", (Hd,)),
        ("mlp.fc2.weight", (D, Ho)), ("mlp.fc2.bias", (D,)),
        *ls[1:],
    ]


def root_param_specs(cfg: ViTConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """Root unit.  The conv weight is stored as a [D, Kpad] GEMM operand (logical [D, 3, P, P]).  The prefix tokens
    (cls_token, reg_token) sit in front of pos_embed, as timm registers them."""
    D = cfg.embed_dim
    prefix = [("cls_token", (1, D))] if cfg.class_token else []
    if cfg.class_token and cfg.reg_tokens:
        prefix.append(("reg_token", (cfg.reg_tokens, D)))
    return [
        ("patch_embed.proj.weight", (D, cfg.patch_kpad)), ("patch_embed.proj.bias", (D,)),
        *prefix,
        ("pos_embed", (cfg.pos_len, D)),
        ("norm.weight", (D,)), ("norm.bias", (D,)),
        ("head.weight", (cfg.num_classes, D)), ("head.bias", (cfg.num_classes,)),
    ]


def logical_shapes(cfg: ViTConfig) -> Dict[str, Tuple[int, ...]]:
    """Shapes a plain timm-style (non-sharded) ViT would have for the stored tensors that differ."""
    P, D = cfg.patch_size, cfg.embed_dim
    out = {"patch_embed.proj.weight": (D, 3, P, P), "pos_embed": (1, cfg.pos_len, D)}
    if cfg.class_token:
        out["cls_token"] = (1, 1, D)
        if cfg.reg_tokens:
            out["reg_token"] = (1, cfg.reg_tokens, D)
    return out


def _linear_init(out_f: int, in_f: int, gen, fan_in: Optional[int] = None, device="cpu"):
    """PyTorch's default nn.Linear / nn.Conv2d init (kaiming_uniform a=sqrt(5)): U(+-1/sqrt(fan_in)).

    The reference calls timm's ``_init_vit_weights`` on composite modules where it matches nothing
    (run_vit_training.py:125,142), so every Linear/Conv keeps this default init.
    """
    fan_in = fan_in or in_f
    bound = 1.0 / math.sqrt(fan_in)
    w = (torch.rand(out_f, in_f, generator=gen, device=device) * 2.0 - 1.0) * bound
    b = (torch.rand(out_f, generator=gen, device=device) * 2.0 - 1.0) * bound
    return w, b


def init_block_params(cfg: ViTConfig, gen, device="cpu") -> Dict[str, torch.Tensor]:
    D, Hd = cfg.embed_dim, cfg.hidden_dim
    p = {"norm1.weight": torch.ones(D, device=device), "norm1.bias": torch.zeros(D, device=device),
         "norm2.weight": torch.ones(D, device=device), "norm2.bias": torch.zeros(D, device=device)}
    p["attn.qkv.weight"], p["attn.qkv.bias"] = _linear_init(3 * D, D, gen, device=device)
    p["attn.proj.weight"], p["attn.proj.bias"] = _linear_init(D, D, gen, device=device)
    p["mlp.fc1.weight"], p["mlp.fc1.bias"] = _linear_init(Hd, D, gen, device=device)
    p["mlp.fc2.weight"], p["mlp.fc2.bias"] = _linear_init(D, cfg.mlp_out_dim, gen, device=device)
    if cfg.qk_norm:  # nn.LayerNorm init: draws nothing, so every other parameter equals the same-seed model's
        hd = cfg.head_dim
        for n in ("q_norm", "k_norm"):
            p[f"attn.{n}.weight"], p[f"attn.{n}.bias"] = torch.ones(hd, device=device), torch.zeros(hd, device=device)
    if cfg.init_values:  # timm LayerScale: init_values * ones(D), no draws either
        p["ls1.gamma"] = torch.full((D,), float(cfg.init_values), device=device)
        p["ls2.gamma"] = torch.full((D,), float(cfg.init_values), device=device)
    return p


def init_root_params(cfg: ViTConfig, gen, device="cpu") -> Dict[str, torch.Tensor]:
    D = cfg.embed_dim
    p = {}
    w, b = _linear_init(D, cfg.patch_k, gen, device=device)
    wp = torch.zeros(D, cfg.patch_kpad, device=device)
    wp[:, : cfg.patch_k] = w
    p["patch_embed.proj.weight"], p["patch_embed.proj.bias"] = wp, b
    pos = torch.empty(cfg.pos_len, D, device=device)
    torch.nn.init.trunc_normal_(pos, std=0.02, generator=gen)  # run_vit_training.py:128
    p["pos_embed"] = pos
    p["norm.weight"], p["norm.bias"] = torch.ones(D, device=device), torch.zeros(D, device=device)
    p["head.weight"], p["head.bias"] = _linear_init(cfg.num_classes, D, gen, device=device)
    if cfg.class_token:  # timm init_weights: normal(std=1e-6), drawn after every other root draw
        p["cls_token"] = torch.nn.init.normal_(torch.empty(1, D, device=device), std=1e-6, generator=gen)
        if cfg.reg_tokens:
            p["reg_token"] = torch.nn.init.normal_(torch.empty(cfg.reg_tokens, D, device=device), std=1e-6,
                                                   generator=gen)
    return p


# ------------------------------------------------------------------------------------------------
# Dropout (reference flags --pos_dropout / --att_dropout / --mlp_dropout, default 0 -> elided)
# ------------------------------------------------------------------------------------------------
class DropoutCtx:
    """Counter-based dropout: the mask of a site is a pure function of (seed, step, site, position) -- a 64-bit key
    handed to ``ops.dropout`` (Philox kernel on the GPU, seeded generator on the CPU) -- so nothing is stored: the
    activation-checkpoint recompute and the backward pass regenerate exactly the mask the first forward used."""

    def __init__(self, seed: int = 0):
        self.seed = seed
        self.step = 0
        self.training = True
        # Global index of this rank's first sample (rank * local batch).  The per-sample masks of stochastic depth are
        # drawn at the global index, so image b of every rank gets its own draw and the masks do not depend on the
        # world size.  (The element-dropout keys above do not depend on the rank.)
        self.sample_offset = 0

    def key(self, site: int) -> int:
        return (((self.seed * 1000003 + self.step) * 1000003 + site) * 0x9E3779B97F4A7C15) & 0x7FFFFFFFFFFFFFFF


# ------------------------------------------------------------------------------------------------
# Batch mixing (--mixup / --cutmix): timm 0.4.12 Mixup, mode 'batch', image b paired with image B-1-b
# ------------------------------------------------------------------------------------------------
Mix = Tuple[float, Optional[Tuple[int, int, int, int]]]  # (lam, CutMix box (yl, yh, xl, xh) or None for Mixup)


def mix_rng(seed: int, step: int, rank: int) -> np.random.Generator:
    """The host generator of one step's mixing draws: a pure function of (seed, step, rank), so a resumed run draws what
    an uninterrupted one would.  Each rank draws for itself and mixes within its own local batch (DeiT's per-rank
    seeding)."""
    return np.random.default_rng([seed & 0xFFFF_FFFF_FFFF_FFFF, step, rank])


def draw_mix(cfg: ViTConfig, rng: np.random.Generator) -> Optional[Mix]:
    """One step's mixing parameters, drawn like timm's ``Mixup._params_per_batch`` and ``cutmix_bbox_and_lam``
    (margin 0, correct_lam=True) on ``cfg.image_size`` square images.  None when the step does not mix (lam == 1,
    which includes a CutMix box of zero area); otherwise ``(lam, None)`` for Mixup or ``(lam, (yl, yh, xl, xh))`` for
    CutMix."""
    if not cfg.mixing:
        return None
    if not rng.random() < cfg.mixup_prob:
        return None
    if cfg.mixup > 0 and cfg.cutmix > 0:
        use_cutmix = rng.random() < cfg.mixup_switch_prob
    else:
        use_cutmix = cfg.cutmix > 0
    alpha = cfg.cutmix if use_cutmix else cfg.mixup
    lam = float(rng.beta(alpha, alpha))
    box = None
    if use_cutmix:
        S = cfg.image_size
        cut = int(S * np.sqrt(1 - lam))
        cy = int(rng.integers(0, S))
        cx = int(rng.integers(0, S))
        yl, yh = int(np.clip(cy - cut // 2, 0, S)), int(np.clip(cy + cut // 2, 0, S))
        xl, xh = int(np.clip(cx - cut // 2, 0, S)), int(np.clip(cx + cut // 2, 0, S))
        lam = 1.0 - (yh - yl) * (xh - xl) / float(S * S)
        box = (yl, yh, xl, xh)
    return None if lam == 1.0 else (lam, box)


@functools.lru_cache(maxsize=None)
def _drop_path_rates(rate: float, depth: int) -> Tuple[float, ...]:
    return tuple(float(r) for r in torch.linspace(0, rate, depth))


def drop_path_rates(cfg: ViTConfig) -> List[float]:
    """Stochastic-depth rate of every block: torch.linspace(0, drop_path_rate, num_blocks), like timm's ViT."""
    return list(_drop_path_rates(float(cfg.drop_path_rate), int(cfg.num_blocks)))


# ------------------------------------------------------------------------------------------------
# Transformer block
# ------------------------------------------------------------------------------------------------
def block_forward(ops, cfg: ViTConfig, p, x, B: int, save, drop: Optional[DropoutCtx] = None,
                  block_idx: int = 0):
    """x: [B*N, D] -> y: [B*N, D].  With save=True also returns the tensors backward needs; save="lean" keeps
    only what a GEMM would have to recompute (x, qkv, attention output, x1, fc1 pre-activation: 10 [T, D] units
    instead of ~17.6) and block_backward re-materialises h1 / P / h2 / gelu(u) with memory-bound kernels.
    save may also be a set of extras to keep on top of the lean set: "P" (attention probabilities),
    "h" (both LayerNorm outputs), "g" (gelu(u)); True == all three.
    With cfg.qk_norm the attention runs on qkn = qk_norm(qkv).  The lean set keeps the un-normalised qkv and the norm's
    fp32 statistics; save=True also keeps qkn (a checkpoint recompute goes straight into the backward, which needs it).
    A forward that saves nothing normalises in place.
    With prefix tokens every image has cfg.num_tokens rows (class and register tokens first); the block is unchanged.
    The tokens per image are x.shape[0] // B: T' = P + K in a training step with patch dropout.
    With cfg.swiglu, u is the packed [T, Hd] fc1 pre-activation [gate | value] and g = silu(gate) * value [T, Hd / 2]."""
    do_save = save is not False and save is not None
    if save is True:
        extras = frozenset(("P", "h", "g"))
    elif not do_save or isinstance(save, str):
        extras = frozenset()
    else:
        extras = frozenset(save)
    N, H, hd = x.shape[0] // B, cfg.num_heads, cfg.head_dim
    pa, pm = cfg.att_dropout, cfg.mlp_dropout
    use_drop = drop is not None and drop.training and (pa > 0 or pm > 0)
    site = block_idx * 8
    # Stochastic depth: per-sample scales (0 or 1 / keep_prob) of the attention and MLP branches, applied as a row scale
    # in the epilogue of the branch's last GEMM.  Regenerated by a checkpoint recompute from the same keys.
    dpath = None
    if drop is not None and drop.training and cfg.drop_path_rate > 0:
        rate = drop_path_rates(cfg)[block_idx]
        if rate > 0:
            dpath = (ops.drop_path_scale(drop.key(site + 4), rate, B, drop.sample_offset, x.device),
                     ops.drop_path_scale(drop.key(site + 5), rate, B, drop.sample_offset, x.device))
    rs_att = dict(row_scale=dpath[0], rows_per_scale=N) if dpath is not None else {}
    rs_mlp = dict(row_scale=dpath[1], rows_per_scale=N) if dpath is not None else {}
    ag = getattr(p, "ag", None) or {}  # weights whose all-gather is fused into the GEMM that consumes them
    h1, m1, r1 = ops.ln_fwd(x, p["norm1.weight"], p["norm1.bias"], BLOCK_LN_EPS)
    qkv = ops.linear_fwd(h1, p["attn.qkv.weight"], p["attn.qkv.bias"], ag=ag.get("attn.qkv.weight"))
    qkn = qkv  # what the attention reads: qkv, or with QK normalisation its normalised copy
    if cfg.qk_norm:
        qkn, qk_mean, qk_rstd = _qk_norm(ops, cfg, p, qkv, inplace=not do_save)
    masks = {}  # site name -> dropout key (the masks themselves are regenerated, never stored)
    lse = None
    if use_drop and pa > 0:
        masks["att"] = drop.key(site + 0)
        if ops.use_flash(N, hd):  # the fused kernels apply the dropout mask in registers
            if do_save:
                a, lse = ops.attention_fwd_lse(qkn, B, N, H, hd, drop=(pa, masks["att"]))
                P = None
            else:
                a, P = ops.attention_fwd(qkn, B, N, H, hd, drop=(pa, masks["att"]), need_p=False)
        else:
            a, P = ops.attention_fwd(qkn, B, N, H, hd, drop=(pa, masks["att"]))
    elif do_save and ops.use_flash(N, hd):
        a, lse = ops.attention_fwd_lse(qkn, B, N, H, hd)  # backward rebuilds P from the row log-sum-exp
        P = None
    else:
        a, P = ops.attention_fwd(qkn, B, N, H, hd, need_p="P" in extras)
    w_proj, b_proj = _branch_layer(ops, cfg, p, "attn.proj", "ls1")
    if use_drop and pm > 0:
        # timm feeds `drop` to both proj_drop and the two MLP dropouts
        masks["proj"] = drop.key(site + 1)
        t = ops.linear_fwd(a, w_proj, b_proj, **rs_att)
        x1 = x + ops.dropout(t, pm, masks["proj"])  # the per-sample row scale commutes with the element mask
    else:
        x1 = ops.linear_fwd(a, w_proj, b_proj, residual=x, **rs_att)
    del w_proj, b_proj
    h2, m2, r2 = ops.ln_fwd(x1, p["norm2.weight"], p["norm2.bias"], BLOCK_LN_EPS)
    act = "swiglu" if cfg.swiglu else "gelu"
    if do_save:
        g, u = ops.linear_fwd(h2, p["mlp.fc1.weight"], p["mlp.fc1.bias"], act=act, want_preact=True,
                              ag=ag.get("mlp.fc1.weight"))
    else:
        g, u = ops.linear_fwd(h2, p["mlp.fc1.weight"], p["mlp.fc1.bias"], act=act, ag=ag.get("mlp.fc1.weight")), None
    w_fc2, b_fc2 = _branch_layer(ops, cfg, p, "mlp.fc2", "ls2")
    if use_drop and pm > 0:
        masks["fc1"] = drop.key(site + 2)
        masks["fc2"] = drop.key(site + 3)
        g = ops.dropout(g, pm, masks["fc1"])
        t = ops.linear_fwd(g, w_fc2, b_fc2, **rs_mlp)
        y = x1 + ops.dropout(t, pm, masks["fc2"])
    else:
        y = ops.linear_fwd(g, w_fc2, b_fc2, residual=x1, **rs_mlp)
    del w_fc2, b_fc2
    if not do_save:
        return y, None
    saved = dict(x=x, m1=m1, r1=r1, qkv=qkv, a=a, x1=x1, m2=m2, r2=r2, u=u, masks=masks, lse=lse)
    if dpath is not None:
        saved["dpath"] = dpath
    if cfg.qk_norm:
        saved["qk_mean"], saved["qk_rstd"] = qk_mean, qk_rstd
        if save is True:
            saved["qkn"] = qkn
    if "P" in extras and lse is None:
        saved["P"] = P
    if "h" in extras:
        saved["h1"], saved["h2"] = h1, h2
    if "g" in extras:
        saved["g"] = g
    return y, saved


def block_backward(ops, cfg: ViTConfig, p, G, s, dy, dy_colsum, B: int):
    """Backward of one block.

    p / G: parameter and gradient views of this unit.  dy_colsum = column sums of dy (fp32), which *is*
    the fc2 bias gradient; it is produced for free by whoever computed dy (the LN backward of the block
    above).  Returns (dx, colsum(dx)) for the block below.
    With LayerScale the proj / fc2 bias gradient is gamma o colsum instead; the wgrad runs first, then
    ``ops.layer_scale_bwd`` rescales its result and yields the bias and gamma gradients, and the dgrad uses the
    folded weight.
    """
    N, H, hd = s["x"].shape[0] // B, cfg.num_heads, cfg.head_dim
    pa, pm = cfg.att_dropout, cfg.mlp_dropout
    masks = s["masks"]
    dpath = s.get("dpath")  # stochastic depth: per-sample scales of the (attention, MLP) branches, or None
    # ---- MLP ----
    if dpath is not None:  # the branch gradient is scaled per sample; the residual gradient dy stays as it is
        dt = ops.dropout(dy, pm, masks["fc2"]) if "fc2" in masks else dy
        dt, s2 = ops.drop_path_bwd(dt, dpath[1], N)
    elif "fc2" in masks:
        dt = ops.dropout(dy, pm, masks["fc2"])
        s2 = ops.colsum(dt)
    else:
        dt = dy
        s2 = dy_colsum
    if not cfg.init_values:
        G["mlp.fc2.bias"].copy_(s2)
    g = s.pop("g", None)
    if g is None:  # not kept: re-materialise from the pre-activation
        g = ops.swiglu_fwd(s["u"]) if cfg.swiglu else ops.gelu_fwd(s["u"])
        if "fc1" in masks:
            g = ops.dropout(g, pm, masks["fc1"])
    ops.linear_wgrad(dt, g, out=G["mlp.fc2.weight"])
    del g
    w_fc2 = _layer_scale_bwd(ops, p, G, "mlp.fc2", "ls2", s2) if cfg.init_values else p["mlp.fc2.weight"]
    if "fc1" in masks:
        dg = ops.dropout(ops.linear_dgrad(dt, w_fc2), pm, masks["fc1"])
        du = ops.swiglu_bwd(dg, s["u"]) if cfg.swiglu else ops.dgelu_mul(dg, s["u"])
        db1 = ops.colsum(du)
    elif cfg.swiglu:
        du, db1 = ops.linear_dgrad(dt, w_fc2, dswiglu_preact=s["u"], want_colsum=True)
    else:
        du, db1 = ops.linear_dgrad(dt, w_fc2, dgelu_preact=s["u"], want_colsum=True)
    del w_fc2
    G["mlp.fc1.bias"].copy_(db1)
    h2 = s.pop("h2", None)
    if h2 is None:
        h2 = ops.ln_fwd(s["x1"], p["norm2.weight"], p["norm2.bias"], BLOCK_LN_EPS)[0]
    ops.linear_wgrad(du, h2, out=G["mlp.fc1.weight"])
    del h2
    dh2 = ops.linear_dgrad(du, p["mlp.fc1.weight"])
    del du
    dx1, dn2w, dn2b, dx1_sum = ops.ln_bwd(dh2, s["x1"], p["norm2.weight"], s["m2"], s["r2"], dres=dy, want_dxsum=True)
    del dh2
    G["norm2.weight"].copy_(dn2w)
    G["norm2.bias"].copy_(dn2b)
    # ---- attention ----
    if dpath is not None:
        dt = ops.dropout(dx1, pm, masks["proj"]) if "proj" in masks else dx1
        dt, s1 = ops.drop_path_bwd(dt, dpath[0], N)
    elif "proj" in masks:
        dt = ops.dropout(dx1, pm, masks["proj"])
        s1 = ops.colsum(dt)
    else:
        dt = dx1
        s1 = dx1_sum
    if not cfg.init_values:
        G["attn.proj.bias"].copy_(s1)
    ops.linear_wgrad(dt, s["a"], out=G["attn.proj.weight"])
    w_proj = _layer_scale_bwd(ops, p, G, "attn.proj", "ls1", s1) if cfg.init_values else p["attn.proj.weight"]
    da = ops.linear_dgrad(dt, w_proj)
    del w_proj
    qkn = s["qkv"]
    if cfg.qk_norm:
        qkn = s.pop("qkn", None)
        if qkn is None:  # not kept: rebuild the normalised copy the attention read
            qkn = _qk_norm(ops, cfg, p, s["qkv"], inplace=False)[0]
    if s.get("lse") is not None:  # flash-style: P (and the dropout mask) is rebuilt inside the fused backward kernels
        dqkv, dbqkv = ops.attention_bwd_lse(da, qkn, s["a"], s["lse"], B, N, H, hd, want_colsum=True,
                                            drop=(pa, masks["att"]) if "att" in masks else None)
    else:
        if s.get("P") is None:
            s["P"] = ops.attention_probs(qkn, B, N, H, hd)
        if "att" in masks:
            dqkv, dbqkv = ops.attention_bwd(da, qkn, s["P"], B, N, H, hd, want_colsum=True,
                                            drop=(pa, masks["att"]))
        else:
            dqkv, dbqkv = ops.attention_bwd(da, qkn, s["P"], B, N, H, hd, want_colsum=True)
    del da, qkn
    if cfg.qk_norm:
        # dq / dk become the gradients of the un-normalised q / k; the bias is added before the norm, so the column
        # sums of the new dq / dk are the q / k part of the qkv bias gradient (dv and its sums are unchanged)
        D = cfg.embed_dim
        _, dwq, dbq, dwk, dbk, cs = ops.qk_norm_bwd(dqkv, s["qkv"], H, hd, p["attn.q_norm.weight"],
                                                    p["attn.k_norm.weight"], s["qk_mean"], s["qk_rstd"])
        dbqkv[: 2 * D].copy_(cs)
        G["attn.q_norm.weight"].copy_(dwq)
        G["attn.q_norm.bias"].copy_(dbq)
        G["attn.k_norm.weight"].copy_(dwk)
        G["attn.k_norm.bias"].copy_(dbk)
    G["attn.qkv.bias"].copy_(dbqkv)
    s["P"] = None
    h1 = s.pop("h1", None)
    if h1 is None:
        h1 = ops.ln_fwd(s["x"], p["norm1.weight"], p["norm1.bias"], BLOCK_LN_EPS)[0]
    ops.linear_wgrad(dqkv, h1, out=G["attn.qkv.weight"])
    del h1
    dh1 = ops.linear_dgrad(dqkv, p["attn.qkv.weight"])
    del dqkv
    dx, dn1w, dn1b, dx_sum = ops.ln_bwd(dh1, s["x"], p["norm1.weight"], s["m1"], s["r1"], dres=dx1, want_dxsum=True)
    G["norm1.weight"].copy_(dn1w)
    G["norm1.bias"].copy_(dn1b)
    return dx, dx_sum


def _branch_layer(ops, cfg: ViTConfig, p, layer: str, ls: str):
    """Weight and bias of a branch's last layer, with LayerScale folded in: (gamma o W, gamma o b)."""
    w, b = p[f"{layer}.weight"], p[f"{layer}.bias"]
    return ops.layer_scale_fold(w, b, p[f"{ls}.gamma"]) if cfg.init_values else (w, b)


def _layer_scale_bwd(ops, p, G, layer: str, ls: str, colsum):
    """After the wgrad has written M = dy'^T a into G[layer.weight]: turns it into dW = gamma o M and writes the bias
    and gamma gradients (colsum = column sums of dy').  Returns the folded weight the dgrad multiplies by."""
    wg, db, dgamma = ops.layer_scale_bwd(p[f"{layer}.weight"], p[f"{layer}.bias"], p[f"{ls}.gamma"],
                                         G[f"{layer}.weight"], colsum)
    G[f"{layer}.bias"].copy_(db)
    G[f"{ls}.gamma"].copy_(dgamma)
    return wg


def _qk_norm(ops, cfg: ViTConfig, p, qkv, inplace: bool):
    return ops.qk_norm_fwd(qkv, cfg.num_heads, cfg.head_dim, p["attn.q_norm.weight"], p["attn.q_norm.bias"],
                           p["attn.k_norm.weight"], p["attn.k_norm.bias"], BLOCK_LN_EPS, inplace=inplace)


# ------------------------------------------------------------------------------------------------
# Stem (patch embed + pos embed) and head (final norm, mean pool, classifier, loss)
# ------------------------------------------------------------------------------------------------
def stem_forward(ops, cfg: ViTConfig, p, images, dtype, drop: Optional[DropoutCtx] = None, mix: Optional[Mix] = None):
    """mix: this step's batch mixing (``draw_mix``), applied inside the im2col; the saved cols are the mixed patches.
    With a class token the patch GEMM adds the patch rows of pos_embed and ops.tokens_fwd puts the prefix tokens in
    front of every image: timm's cat(prefix, patches) + pos, or cat(prefix, patches + pos) with no_embed_class.
    With patch dropout in training (``_stem_forward_patch_drop``) every image keeps cfg.num_keep patches."""
    B = images.shape[0]
    if drop is not None and drop.training and cfg.patch_drop_rate > 0:
        x0, saved = _stem_forward_patch_drop(ops, cfg, p, images, dtype, drop, mix)
    else:
        if mix is None:
            cols = ops.patch_im2col(images, cfg.patch_size, cfg.patch_kpad, dtype)
        else:
            cols = ops.patch_im2col(images, cfg.patch_size, cfg.patch_kpad, dtype, mix=mix)
        if cfg.class_token:
            P, pos = cfg.num_prefix_tokens, p["pos_embed"]
            y = ops.linear_fwd(cols, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"],
                               residual=pos if cfg.no_embed_class else pos[P:], res_row_mod=cfg.num_patches)
            x0 = ops.tokens_fwd(y, p["cls_token"], p.get("reg_token"), None if cfg.no_embed_class else pos[:P], B,
                                cfg.num_patches)
            del y
        else:
            x0 = ops.linear_fwd(cols, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"],
                                residual=p["pos_embed"], res_row_mod=cfg.num_patches)
        saved = dict(cols=cols)
    mask = None  # dropout key of the position-embedding dropout (reference :129,157)
    if drop is not None and drop.training and cfg.pos_dropout > 0:
        mask = drop.key(7_000_001)
        x0 = ops.dropout(x0, cfg.pos_dropout, mask)
    return x0, dict(saved, mask=mask, B=B)


def _stem_forward_patch_drop(ops, cfg: ViTConfig, p, images, dtype, drop: DropoutCtx, mix: Optional[Mix]):
    """timm PatchDropout(ordered=True) after the position embedding: image g = drop.sample_offset + b keeps the
    patches ops.patch_drop_select draws for it (key 7_000_002), in ascending order.  Only the kept patches go through
    the im2col and the patch GEMM, which adds the bias and their own pos_embed rows (ops.pos_gather) as its residual;
    the prefix tokens are always kept.  pos_drop then acts on the compacted [B * (P + K), D] buffer."""
    B, N, K, P = images.shape[0], cfg.num_patches, cfg.num_keep, cfg.num_prefix_tokens
    keep, inv = ops.patch_drop_select(drop.key(7_000_002), B, N, K, drop.sample_offset, images.device)
    if mix is None:
        cols = ops.patch_im2col(images, cfg.patch_size, cfg.patch_kpad, dtype, keep=keep)
    else:
        cols = ops.patch_im2col(images, cfg.patch_size, cfg.patch_kpad, dtype, mix=mix, keep=keep)
    pos = p["pos_embed"]
    pos_patch = pos[P:] if cfg.class_token and not cfg.no_embed_class else pos
    x0 = ops.linear_fwd(cols, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"],
                        residual=ops.pos_gather(pos_patch, keep))
    if cfg.class_token:
        x0 = ops.tokens_fwd(x0, p["cls_token"], p.get("reg_token"), None if cfg.no_embed_class else pos[:P], B, K)
    return x0, dict(cols=cols, keep=keep, inv=inv)


def stem_backward(ops, cfg: ViTConfig, p, G, s, dx0, dx0_colsum):
    if s.get("inv") is not None:
        _stem_backward_patch_drop(ops, cfg, G, s, dx0)
        return
    if cfg.class_token:
        _stem_backward_prefix(ops, cfg, G, s, dx0)
        return
    if s["mask"] is not None:
        dx0 = ops.dropout(dx0, cfg.pos_dropout, s["mask"])
        dx0_colsum = ops.colsum(dx0)
    ops.linear_wgrad(dx0, s["cols"], out=G["patch_embed.proj.weight"])
    G["patch_embed.proj.bias"].copy_(dx0_colsum)
    G["pos_embed"].copy_(dx0.view(s["B"], cfg.num_patches, cfg.embed_dim).sum(dim=0, dtype=torch.float32))


def _stem_backward_patch_drop(ops, cfg: ViTConfig, G, s, dx0):
    """With patch dropout: one pass (ops.patch_drop_bwd) scatters dx0 [B * (P + K), D] back to the full sequence as
    per-token batch sums dtok [P + N, D] (a dropped patch gets nothing from that image) and, with prefix tokens, copies
    the patch rows out as the wgrad operand; without them dx0 itself is that operand."""
    if s["mask"] is not None:
        dx0 = ops.dropout(dx0, cfg.pos_dropout, s["mask"])
    P = cfg.num_prefix_tokens
    dpatch, dtok = ops.patch_drop_bwd(dx0, s["inv"], s["B"], cfg.num_patches, cfg.num_keep, P)
    ops.linear_wgrad(dpatch if P else dx0, s["cols"], out=G["patch_embed.proj.weight"])
    del dpatch
    G["patch_embed.proj.bias"].copy_(dtok[P:].sum(dim=0))
    G["pos_embed"].copy_(dtok[P:] if cfg.no_embed_class else dtok)
    if cfg.class_token:
        G["cls_token"].copy_(dtok[:1])
        if cfg.reg_tokens:
            G["reg_token"].copy_(dtok[1:P])


def _stem_backward_prefix(ops, cfg: ViTConfig, G, s, dx0):
    """With prefix tokens: one pass (ops.tokens_bwd) splits dx0 into the patch rows, the wgrad operand, and the
    per-token batch sums dtok [T, D], which hold the cls / reg / pos_embed gradients and, summed over the patch rows,
    the patch bias gradient (the block-0 column sum would include the prefix rows)."""
    if s["mask"] is not None:
        dx0 = ops.dropout(dx0, cfg.pos_dropout, s["mask"])
    P = cfg.num_prefix_tokens
    dpatch, dtok = ops.tokens_bwd(dx0, s["B"], cfg.num_patches, P)
    ops.linear_wgrad(dpatch, s["cols"], out=G["patch_embed.proj.weight"])
    del dpatch
    G["patch_embed.proj.bias"].copy_(dtok[P:].sum(dim=0))
    G["pos_embed"].copy_(dtok[P:] if cfg.no_embed_class else dtok)
    G["cls_token"].copy_(dtok[:1])
    if cfg.reg_tokens:
        G["reg_token"].copy_(dtok[1:P])


def head_forward(ops, cfg: ViTConfig, p, x, B: int):
    """logits = head(mean_tokens(norm(x)))   (run_vit_training.py:161)
    With a class token: logits = head(norm(x)[:, 0]); the norm acts per row, so only the B class rows are normalised."""
    T = x.shape[0] // B  # cfg.num_tokens, or P + K in a training step with patch dropout
    if cfg.class_token:
        xc = x.view(B, T, cfg.embed_dim)[:, 0].contiguous()
        xn, m, r = ops.ln_fwd(xc, p["norm.weight"], p["norm.bias"], FINAL_LN_EPS)
        logits = ops.linear_fwd(xn, p["head.weight"], p["head.bias"])
        return logits, dict(x=xc, m=m, r=r, pooled=xn, T=T)
    xn, m, r = ops.ln_fwd(x, p["norm.weight"], p["norm.bias"], FINAL_LN_EPS)
    pooled = ops.mean_pool(xn, B, T)  # the mean over the patches present: timm's x[:, P:].mean(1) with P = 0
    logits = ops.linear_fwd(pooled, p["head.weight"], p["head.bias"])
    return logits, dict(x=x, m=m, r=r, pooled=pooled)


def head_backward(ops, cfg: ViTConfig, p, G, s, dlogits, B: int):
    D = cfg.embed_dim
    ops.linear_wgrad(dlogits, s["pooled"], out=G["head.weight"])
    G["head.bias"].copy_(dlogits.sum(dim=0, dtype=torch.float32))
    dpooled = ops.linear_dgrad(dlogits, p["head.weight"])
    if cfg.class_token:  # the LayerNorm backward of the B class rows, placed at token 0 of a zero [B*T, D] gradient
        dxc, dnw, dnb, dx_sum = ops.ln_bwd(dpooled, s["x"], p["norm.weight"], s["m"], s["r"], want_dxsum=True)
        G["norm.weight"].copy_(dnw)
        G["norm.bias"].copy_(dnb)
        dx = torch.zeros(B * s["T"], D, dtype=dxc.dtype, device=dxc.device)
        dx.view(B, s["T"], D)[:, 0] = dxc
        return dx, dx_sum
    dxn = ops.mean_pool_bwd(dpooled, B, s["x"].shape[0] // B)
    dx, dnw, dnb, dx_sum = ops.ln_bwd(dxn, s["x"], p["norm.weight"], s["m"], s["r"], want_dxsum=True)
    G["norm.weight"].copy_(dnw)
    G["norm.bias"].copy_(dnb)
    return dx, dx_sum
