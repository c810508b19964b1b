"""Vision Transformer as an explicit functional graph with hand-written forward *and* backward.

Architecture parity with the reference model (run_vit_training.py:99-162, timm 0.4.12 blocks):
  * PatchEmbed = Conv2d(3, D, k=s=P) -> tokens; learned pos_embed; dropout           (:124-129,156-157)
  * num_blocks pre-LN blocks: x += proj(attn(norm1(x))); x += fc2(gelu(fc1(norm2(x))))  (:133-141)
    - LayerNorm eps 1e-5 inside blocks, qkv_bias=True, exact (erf) GELU
    - optional stochastic depth (timm drop_path, off in the reference): x += drop_path(branch) for both branches,
      one Bernoulli per sample and branch, kept samples scaled by 1 / keep_prob, block i at rate
      linspace(0, drop_path_rate, num_blocks)[i], nothing dropped in eval
  * optional Mixup / CutMix (timm Mixup, mode 'batch', off in the reference): drawn on the host per step (draw_mix),
    applied inside the patch im2col, with the mixed, smoothed target handled by the cross-entropy
  * final LayerNorm(eps=1e-6), mean-pool over tokens (no CLS token), Linear head      (:151-153,159-161)
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
    D, Hd = cfg.embed_dim, cfg.hidden_dim
    return [
        ("norm1.weight", (D,)), ("norm1.bias", (D,)),
        ("attn.qkv.weight", (3 * D, D)), ("attn.qkv.bias", (3 * D,)),
        ("attn.proj.weight", (D, D)), ("attn.proj.bias", (D,)),
        ("norm2.weight", (D,)), ("norm2.bias", (D,)),
        ("mlp.fc1.weight", (Hd, D)), ("mlp.fc1.bias", (Hd,)),
        ("mlp.fc2.weight", (D, Hd)), ("mlp.fc2.bias", (D,)),
    ]


def root_param_specs(cfg: ViTConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """Root unit.  The conv weight is stored as a [D, Kpad] GEMM operand (logical [D, 3, P, P])."""
    D = cfg.embed_dim
    return [
        ("patch_embed.proj.weight", (D, cfg.patch_kpad)), ("patch_embed.proj.bias", (D,)),
        ("pos_embed", (cfg.num_patches, D)),
        ("norm.weight", (D,)), ("norm.bias", (D,)),
        ("head.weight", (cfg.num_classes, D)), ("head.bias", (cfg.num_classes,)),
    ]


def logical_shapes(cfg: ViTConfig) -> Dict[str, Tuple[int, ...]]:
    """Shapes a plain timm-style (non-sharded) ViT would have for the stored tensors that differ."""
    P = cfg.patch_size
    return {"patch_embed.proj.weight": (cfg.embed_dim, 3, P, P), "pos_embed": (1, cfg.num_patches, cfg.embed_dim)}


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
    p["mlp.fc2.weight"], p["mlp.fc2.bias"] = _linear_init(D, Hd, gen, device=device)
    return p


def init_root_params(cfg: ViTConfig, gen, device="cpu") -> Dict[str, torch.Tensor]:
    D = cfg.embed_dim
    p = {}
    w, b = _linear_init(D, cfg.patch_k, gen, device=device)
    wp = torch.zeros(D, cfg.patch_kpad, device=device)
    wp[:, : cfg.patch_k] = w
    p["patch_embed.proj.weight"], p["patch_embed.proj.bias"] = wp, b
    pos = torch.empty(cfg.num_patches, D, device=device)
    torch.nn.init.trunc_normal_(pos, std=0.02, generator=gen)  # run_vit_training.py:128
    p["pos_embed"] = pos
    p["norm.weight"], p["norm.bias"] = torch.ones(D, device=device), torch.zeros(D, device=device)
    p["head.weight"], p["head.bias"] = _linear_init(cfg.num_classes, D, gen, device=device)
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
    "h" (both LayerNorm outputs), "g" (gelu(u)); True == all three."""
    do_save = save is not False and save is not None
    if save is True:
        extras = frozenset(("P", "h", "g"))
    elif not do_save or isinstance(save, str):
        extras = frozenset()
    else:
        extras = frozenset(save)
    N, H, hd = cfg.num_patches, cfg.num_heads, cfg.head_dim
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
    masks = {}  # site name -> dropout key (the masks themselves are regenerated, never stored)
    lse = None
    if use_drop and pa > 0:
        masks["att"] = drop.key(site + 0)
        if ops.use_flash(N, hd):  # the fused kernels apply the dropout mask in registers
            if do_save:
                a, lse = ops.attention_fwd_lse(qkv, B, N, H, hd, drop=(pa, masks["att"]))
                P = None
            else:
                a, P = ops.attention_fwd(qkv, B, N, H, hd, drop=(pa, masks["att"]), need_p=False)
        else:
            a, P = ops.attention_fwd(qkv, B, N, H, hd, drop=(pa, masks["att"]))
    elif do_save and ops.use_flash(N, hd):
        a, lse = ops.attention_fwd_lse(qkv, B, N, H, hd)  # backward rebuilds P from the row log-sum-exp
        P = None
    else:
        a, P = ops.attention_fwd(qkv, B, N, H, hd, need_p="P" in extras)
    if use_drop and pm > 0:
        # timm feeds `drop` to both proj_drop and the two MLP dropouts
        masks["proj"] = drop.key(site + 1)
        t = ops.linear_fwd(a, p["attn.proj.weight"], p["attn.proj.bias"], **rs_att)
        x1 = x + ops.dropout(t, pm, masks["proj"])  # the per-sample row scale commutes with the element mask
    else:
        x1 = ops.linear_fwd(a, p["attn.proj.weight"], p["attn.proj.bias"], residual=x, **rs_att)
    h2, m2, r2 = ops.ln_fwd(x1, p["norm2.weight"], p["norm2.bias"], BLOCK_LN_EPS)
    if do_save:
        g, u = ops.linear_fwd(h2, p["mlp.fc1.weight"], p["mlp.fc1.bias"], act="gelu", want_preact=True,
                              ag=ag.get("mlp.fc1.weight"))
    else:
        g, u = ops.linear_fwd(h2, p["mlp.fc1.weight"], p["mlp.fc1.bias"], act="gelu", ag=ag.get("mlp.fc1.weight")), None
    if use_drop and pm > 0:
        masks["fc1"] = drop.key(site + 2)
        masks["fc2"] = drop.key(site + 3)
        g = ops.dropout(g, pm, masks["fc1"])
        t = ops.linear_fwd(g, p["mlp.fc2.weight"], p["mlp.fc2.bias"], **rs_mlp)
        y = x1 + ops.dropout(t, pm, masks["fc2"])
    else:
        y = ops.linear_fwd(g, p["mlp.fc2.weight"], p["mlp.fc2.bias"], residual=x1, **rs_mlp)
    if not do_save:
        return y, None
    saved = dict(x=x, m1=m1, r1=r1, qkv=qkv, a=a, x1=x1, m2=m2, r2=r2, u=u, masks=masks, lse=lse)
    if dpath is not None:
        saved["dpath"] = dpath
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
    """
    N, H, hd = cfg.num_patches, cfg.num_heads, cfg.head_dim
    pa, pm = cfg.att_dropout, cfg.mlp_dropout
    masks = s["masks"]
    dpath = s.get("dpath")  # stochastic depth: per-sample scales of the (attention, MLP) branches, or None
    # ---- MLP ----
    if dpath is not None:  # the branch gradient is scaled per sample; the residual gradient dy stays as it is
        dt = ops.dropout(dy, pm, masks["fc2"]) if "fc2" in masks else dy
        dt, db2 = ops.drop_path_bwd(dt, dpath[1], N)
        G["mlp.fc2.bias"].copy_(db2)
    elif "fc2" in masks:
        dt = ops.dropout(dy, pm, masks["fc2"])
        G["mlp.fc2.bias"].copy_(ops.colsum(dt))
    else:
        dt = dy
        G["mlp.fc2.bias"].copy_(dy_colsum)
    g = s.pop("g", None)
    if g is None:  # not kept: re-materialise from the pre-activation
        g = ops.gelu_fwd(s["u"])
        if "fc1" in masks:
            g = ops.dropout(g, pm, masks["fc1"])
    ops.linear_wgrad(dt, g, out=G["mlp.fc2.weight"])
    del g
    if "fc1" in masks:
        dg = ops.dropout(ops.linear_dgrad(dt, p["mlp.fc2.weight"]), pm, masks["fc1"])
        du = ops.dgelu_mul(dg, s["u"])
        db1 = ops.colsum(du)
    else:
        du, db1 = ops.linear_dgrad(dt, p["mlp.fc2.weight"], dgelu_preact=s["u"], want_colsum=True)
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
        dt, dbp = ops.drop_path_bwd(dt, dpath[0], N)
        G["attn.proj.bias"].copy_(dbp)
    elif "proj" in masks:
        dt = ops.dropout(dx1, pm, masks["proj"])
        G["attn.proj.bias"].copy_(ops.colsum(dt))
    else:
        dt = dx1
        G["attn.proj.bias"].copy_(dx1_sum)
    ops.linear_wgrad(dt, s["a"], out=G["attn.proj.weight"])
    da = ops.linear_dgrad(dt, p["attn.proj.weight"])
    if s.get("lse") is not None:  # flash-style: P (and the dropout mask) is rebuilt inside the fused backward kernels
        dqkv, dbqkv = ops.attention_bwd_lse(da, s["qkv"], s["a"], s["lse"], B, N, H, hd, want_colsum=True,
                                            drop=(pa, masks["att"]) if "att" in masks else None)
    else:
        if s.get("P") is None:
            s["P"] = ops.attention_probs(s["qkv"], B, N, H, hd)
        if "att" in masks:
            dqkv, dbqkv = ops.attention_bwd(da, s["qkv"], s["P"], B, N, H, hd, want_colsum=True,
                                            drop=(pa, masks["att"]))
        else:
            dqkv, dbqkv = ops.attention_bwd(da, s["qkv"], s["P"], B, N, H, hd, want_colsum=True)
    del da
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


# ------------------------------------------------------------------------------------------------
# Stem (patch embed + pos embed) and head (final norm, mean pool, classifier, loss)
# ------------------------------------------------------------------------------------------------
def stem_forward(ops, cfg: ViTConfig, p, images, dtype, drop: Optional[DropoutCtx] = None, mix: Optional[Mix] = None):
    """mix: this step's batch mixing (``draw_mix``), applied inside the im2col; the saved cols are the mixed patches."""
    B = images.shape[0]
    if mix is None:
        cols = ops.patch_im2col(images, cfg.patch_size, cfg.patch_kpad, dtype)
    else:
        cols = ops.patch_im2col(images, cfg.patch_size, cfg.patch_kpad, dtype, mix=mix)
    x0 = ops.linear_fwd(cols, p["patch_embed.proj.weight"], p["patch_embed.proj.bias"], residual=p["pos_embed"],
                        res_row_mod=cfg.num_patches)
    mask = None  # dropout key of the position-embedding dropout (reference :129,157)
    if drop is not None and drop.training and cfg.pos_dropout > 0:
        mask = drop.key(7_000_001)
        x0 = ops.dropout(x0, cfg.pos_dropout, mask)
    return x0, dict(cols=cols, mask=mask, B=B)


def stem_backward(ops, cfg: ViTConfig, p, G, s, dx0, dx0_colsum):
    if s["mask"] is not None:
        dx0 = ops.dropout(dx0, cfg.pos_dropout, s["mask"])
        dx0_colsum = ops.colsum(dx0)
    ops.linear_wgrad(dx0, s["cols"], out=G["patch_embed.proj.weight"])
    G["patch_embed.proj.bias"].copy_(dx0_colsum)
    G["pos_embed"].copy_(dx0.view(s["B"], cfg.num_patches, cfg.embed_dim).sum(dim=0, dtype=torch.float32))


def head_forward(ops, cfg: ViTConfig, p, x, B: int):
    """logits = head(mean_tokens(norm(x)))   (run_vit_training.py:161)"""
    N, D = cfg.num_patches, cfg.embed_dim
    xn, m, r = ops.ln_fwd(x, p["norm.weight"], p["norm.bias"], FINAL_LN_EPS)
    pooled = ops.mean_pool(xn, B, N)
    logits = ops.linear_fwd(pooled, p["head.weight"], p["head.bias"])
    return logits, dict(x=x, m=m, r=r, pooled=pooled)


def head_backward(ops, cfg: ViTConfig, p, G, s, dlogits, B: int):
    N, D = cfg.num_patches, cfg.embed_dim
    ops.linear_wgrad(dlogits, s["pooled"], out=G["head.weight"])
    G["head.bias"].copy_(dlogits.sum(dim=0, dtype=torch.float32))
    dpooled = ops.linear_dgrad(dlogits, p["head.weight"])
    dxn = ops.mean_pool_bwd(dpooled, B, N)
    dx, dnw, dnb, dx_sum = ops.ln_bwd(dxn, s["x"], p["norm.weight"], s["m"], s["r"], want_dxsum=True)
    G["norm.weight"].copy_(dnw)
    G["norm.bias"].copy_(dnb)
    return dx, dx_sum
