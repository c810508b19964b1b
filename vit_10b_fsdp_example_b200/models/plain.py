"""A plain (un-sharded, autograd) ``nn.Module`` ViT with timm-compatible parameter names.

This is the consumer side of the checkpoint contract: the reference's per-rank files exist so that an offline tool
can rebuild a full ``state_dict`` "loadable into a plain (non-FSDP) ViT" (utils.py:27-28).
``PlainViT.load_state_dict(consolidated, strict=True)`` accepts exactly what ``consolidate_sharded_ckpts`` writes.
The architecture is the reference's FSDPViTModel (run_vit_training.py:99-162) without the wrappers: conv patch embed,
learned position embedding, pre-LN blocks (LayerNorm eps 1e-5), final LayerNorm (eps 1e-6), mean pool, linear head.
It runs on stock PyTorch ops (any device) and is meant for evaluation / export / fine-tuning outside the engine.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..config import ViTConfig


class _Attention(nn.Module):
    def __init__(self, dim: int, num_heads: int, attn_drop: float, proj_drop: float):
        super().__init__()
        self.num_heads = num_heads
        self.qkv = nn.Linear(dim, 3 * dim, bias=True)
        self.attn_drop = attn_drop
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)

    def forward(self, x):
        B, N, C = x.shape
        q, k, v = self.qkv(x).reshape(B, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        o = F.scaled_dot_product_attention(q, k, v, dropout_p=self.attn_drop if self.training else 0.0)
        return self.proj_drop(self.proj(o.transpose(1, 2).reshape(B, N, C)))


class _Mlp(nn.Module):
    def __init__(self, dim: int, hidden: int, drop: float):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden, dim)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        return self.drop(self.fc2(self.drop(self.act(self.fc1(x)))))


class _Block(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        self.norm1 = nn.LayerNorm(cfg.embed_dim, eps=1e-5)
        self.attn = _Attention(cfg.embed_dim, cfg.num_heads, cfg.att_dropout, cfg.mlp_dropout)
        self.norm2 = nn.LayerNorm(cfg.embed_dim, eps=1e-5)
        self.mlp = _Mlp(cfg.embed_dim, cfg.hidden_dim, cfg.mlp_dropout)

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


class _PatchEmbed(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        self.proj = nn.Conv2d(3, cfg.embed_dim, kernel_size=cfg.patch_size, stride=cfg.patch_size)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class PlainViT(nn.Module):
    def __init__(self, cfg: ViTConfig):
        super().__init__()
        self.cfg = cfg
        self.patch_embed = _PatchEmbed(cfg)
        self.pos_embed = nn.Parameter(torch.zeros(1, cfg.num_patches, cfg.embed_dim))
        self.pos_drop = nn.Dropout(cfg.pos_dropout)
        self.blocks = nn.Sequential(*[_Block(cfg) for _ in range(cfg.num_blocks)])
        self.norm = nn.LayerNorm(cfg.embed_dim, eps=1e-6)
        self.head = nn.Linear(cfg.embed_dim, cfg.num_classes)

    def forward(self, image):
        x = self.pos_drop(self.patch_embed(image) + self.pos_embed)
        x = self.blocks(x)
        return self.head(self.norm(x).mean(dim=1))

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
