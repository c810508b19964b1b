"""A plain (un-sharded, autograd) ``nn.Module`` ViT with timm-compatible parameter names.

This is the consumer side of the checkpoint contract: the reference's per-rank files exist so that an offline tool
can rebuild a full ``state_dict`` "loadable into a plain (non-FSDP) ViT" (utils.py:27-28).
``PlainViT.load_state_dict(consolidated, strict=True)`` accepts exactly what ``consolidate_sharded_ckpts`` writes.
The architecture is the reference's FSDPViTModel (run_vit_training.py:99-162) without the wrappers: conv patch embed,
learned position embedding, pre-LN blocks (LayerNorm eps 1e-5, optionally on q and k per head: ``cfg.qk_norm``;
optionally LayerScale on both branches: ``cfg.init_values``; optionally a SwiGLU MLP: ``cfg.swiglu``), final
LayerNorm (eps 1e-6), mean pool, linear head.
With ``cfg.class_token`` it is timm's token layout instead: ``cls_token`` and ``reg_token`` in front of the patches,
``pos_embed`` over all tokens (or the patches only, ``cfg.no_embed_class``), and the head on token 0.
With ``cfg.patch_drop_rate`` it applies timm's ``PatchDropout(ordered=True)`` after ``pos_drop`` in training.
With ``cfg.rope`` the attention rotates q and k of the patch tokens after ``q_norm`` / ``k_norm`` (EVA-02's 2-D axial
RoPE, ``vit.rope_tables``), each kept patch at its original position.
It runs on stock PyTorch ops (any device) and is meant for evaluation / export / fine-tuning outside the engine.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..config import ViTConfig


class _Attention(nn.Module):
    def __init__(self, dim: int, num_heads: int, attn_drop: float, proj_drop: float, qk_norm: bool = False):
        super().__init__()
        self.num_heads = num_heads
        self.qkv = nn.Linear(dim, 3 * dim, bias=True)
        if qk_norm:  # timm Attention(qk_norm=True): LayerNorm over the head dim of q and k
            self.q_norm = nn.LayerNorm(dim // num_heads, eps=1e-5)
            self.k_norm = nn.LayerNorm(dim // num_heads, eps=1e-5)
        else:
            self.q_norm = self.k_norm = None
        self.attn_drop = attn_drop
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)

    def forward(self, x, rope=None):
        """rope: (cos, sin, P) with cos / sin [B or 1, N - P, hd / 2], the angles of the patch tokens."""
        B, N, C = x.shape
        q, k, v = self.qkv(x).reshape(B, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        if self.q_norm is not None:
            q, k = self.q_norm(q), self.k_norm(k)
        if rope is not None:
            q, k = _rotate(q, *rope), _rotate(k, *rope)
        o = F.scaled_dot_product_attention(q, k, v, dropout_p=self.attn_drop if self.training else 0.0)
        return self.proj_drop(self.proj(o.transpose(1, 2).reshape(B, N, C)))


def _rotate(x, cos, sin, P: int):
    """x [B, H, N, hd]: the interleaved pairs (2i, 2i + 1) of tokens P.. turn by the angles of cos / sin."""
    c, s = cos.unsqueeze(1).to(x.dtype), sin.unsqueeze(1).to(x.dtype)  # [B or 1, 1, N - P, hd / 2]
    xp = x[:, :, P:].unflatten(-1, (-1, 2))
    x0, x1 = xp[..., 0], xp[..., 1]
    y = torch.stack((x0 * c - x1 * s, x1 * c + x0 * s), dim=-1).flatten(-2)
    return torch.cat((x[:, :, :P], y), dim=2)


class _Mlp(nn.Module):
    def __init__(self, dim: int, hidden: int, drop: float):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden, dim)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        return self.drop(self.fc2(self.drop(self.act(self.fc1(x)))))


class _GluMlp(nn.Module):
    """timm GluMlp(act_layer=nn.SiLU, gate_last=False), i.e. SwiGLUPacked: fc1 -> [gate | value], silu(gate) * value,
    drop1, norm (Identity), fc2, drop2."""

    def __init__(self, dim: int, hidden: int, drop: float):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.SiLU()
        self.drop1 = nn.Dropout(drop)
        self.norm = nn.Identity()
        self.fc2 = nn.Linear(hidden // 2, dim)
        self.drop2 = nn.Dropout(drop)

    def forward(self, x):
        gate, value = self.fc1(x).chunk(2, dim=-1)
        return self.drop2(self.fc2(self.norm(self.drop1(self.act(gate) * value))))


class _LayerScale(nn.Module):
    """timm LayerScale: x * gamma, gamma [dim] starting at init_values."""

    def __init__(self, dim: int, init_values: float):
        super().__init__()
        self.gamma = nn.Parameter(init_values * torch.ones(dim))

    def forward(self, x):
        return x * self.gamma


class _Block(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        self.norm1 = nn.LayerNorm(cfg.embed_dim, eps=1e-5)
        self.attn = _Attention(cfg.embed_dim, cfg.num_heads, cfg.att_dropout, cfg.mlp_dropout, cfg.qk_norm)
        self.ls1 = _LayerScale(cfg.embed_dim, cfg.init_values) if cfg.init_values else nn.Identity()
        self.norm2 = nn.LayerNorm(cfg.embed_dim, eps=1e-5)
        self.mlp = (_GluMlp if cfg.swiglu else _Mlp)(cfg.embed_dim, cfg.hidden_dim, cfg.mlp_dropout)
        self.ls2 = _LayerScale(cfg.embed_dim, cfg.init_values) if cfg.init_values else nn.Identity()

    def forward(self, x, rope=None):
        x = x + self.ls1(self.attn(self.norm1(x), rope))
        return x + self.ls2(self.mlp(self.norm2(x)))


class _PatchEmbed(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        self.proj = nn.Conv2d(3, cfg.embed_dim, kernel_size=cfg.patch_size, stride=cfg.patch_size)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class _PatchDropout(nn.Module):
    """timm PatchDropout(prob, num_prefix_tokens, ordered=True): in training every image keeps
    K = max(1, int(N * (1 - prob))) of its N patch tokens, in ascending order, and all prefix tokens.  ``keep`` [B, K]
    pins the subset (the default draws timm's random one)."""

    def __init__(self, prob: float, num_prefix_tokens: int):
        super().__init__()
        self.prob, self.num_prefix_tokens = prob, num_prefix_tokens

    def draw(self, B: int, L: int, device):
        """timm's random subset: [B, K] kept patches, ascending."""
        num_keep = max(1, int(L * (1.0 - self.prob)))
        return torch.argsort(torch.randn(B, L, device=device), dim=-1)[:, :num_keep].sort(dim=-1)[0]

    def forward(self, x, keep=None):
        if not self.training or self.prob == 0.0:
            return x
        P = self.num_prefix_tokens
        prefix, x = x[:, :P], x[:, P:]
        B, L = x.shape[:2]
        if keep is None:
            keep = self.draw(B, L, x.device)
        x = x.gather(1, keep.long().unsqueeze(-1).expand(-1, -1, x.shape[-1]))
        return torch.cat((prefix, x), dim=1) if P else x


class PlainViT(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        self.cfg = cfg
        self.patch_embed = _PatchEmbed(cfg)
        D = cfg.embed_dim
        self.cls_token = nn.Parameter(torch.zeros(1, 1, D)) if cfg.class_token else None
        self.reg_token = nn.Parameter(torch.zeros(1, cfg.reg_tokens, D)) if cfg.class_token and cfg.reg_tokens else None
        self.pos_embed = nn.Parameter(torch.zeros(1, cfg.pos_len, D))
        self.pos_drop = nn.Dropout(cfg.pos_dropout)
        self.patch_drop = _PatchDropout(cfg.patch_drop_rate, cfg.num_prefix_tokens)
        self.blocks = nn.Sequential(*[_Block(cfg) for _ in range(cfg.num_blocks)])
        self.norm = nn.LayerNorm(cfg.embed_dim, eps=1e-6)
        self.head = nn.Linear(cfg.embed_dim, cfg.num_classes)
        if cfg.rope:  # no parameters: buffers kept out of the state_dict
            from .vit import rope_tables
            cos, sin = rope_tables(cfg.grid, cfg.head_dim, cfg.rope_theta, cfg.rope_ref_grid)
            self.register_buffer("rope_cos", cos, persistent=False)
            self.register_buffer("rope_sin", sin, persistent=False)

    def _rope(self, patch_keep):
        """(cos, sin, P) of the patch tokens the blocks see: the full grid, or the kept patches' rows."""
        if not self.cfg.rope:
            return None
        cos, sin = self.rope_cos[None], self.rope_sin[None]
        if patch_keep is not None and self.training and self.cfg.patch_drop_rate > 0:
            idx = patch_keep.long()
            cos, sin = self.rope_cos[idx], self.rope_sin[idx]
        return cos, sin, self.cfg.num_prefix_tokens

    def _blocks(self, x, patch_keep):
        rope = self._rope(patch_keep)
        if rope is None:
            return self.blocks(x)
        for blk in self.blocks:
            x = blk(x, rope)
        return x

    def forward(self, image, patch_keep=None):
        """patch_keep: optional [B, K] kept patches of the patch dropout (training only)."""
        if self.cfg.rope and patch_keep is None and self.training and self.cfg.patch_drop_rate > 0:
            patch_keep = self.patch_drop.draw(image.shape[0], self.cfg.num_patches, image.device)  # RoPE needs them
        if self.cls_token is None:
            x = self.patch_drop(self.pos_drop(self.patch_embed(image) + self.pos_embed), patch_keep)
            x = self._blocks(x, patch_keep)
            return self.head(self.norm(x).mean(dim=1))
        x = self.patch_embed(image)
        prefix = [self.cls_token.expand(x.shape[0], -1, -1)]
        if self.reg_token is not None:
            prefix.append(self.reg_token.expand(x.shape[0], -1, -1))
        if self.cfg.no_embed_class:  # timm _pos_embed: cat(prefix, x + pos) or cat(prefix, x) + pos
            x = torch.cat(prefix + [x + self.pos_embed], dim=1)
        else:
            x = torch.cat(prefix + [x], dim=1) + self.pos_embed
        x = self._blocks(self.patch_drop(self.pos_drop(x), patch_keep), patch_keep)
        return self.head(self.norm(x)[:, 0])

    @classmethod
    def from_consolidated(cls, path_or_state, cfg: ViTConfig) -> "PlainViT":
        """Build from the file / dict written by ``consolidate_sharded_ckpts``."""
        sd = path_or_state
        if not isinstance(sd, dict):
            sd = torch.load(sd, map_location="cpu", weights_only=False)
        sd = sd.get("model", sd)
        m = cls(cfg)
        m.load_state_dict(sd, strict=True)
        return m
