"""Command-line / configuration surface.

The 29 flags of the reference (run_vit_training.py:327-363) are accepted verbatim with the same
defaults (ViT-10B recipe).  H100-specific extras are optional and default to reference behaviour.
"""
from __future__ import annotations

import argparse
from dataclasses import dataclass


def build_arg_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="H100-native FSDP ViT training")
    # ---- reference flags (run_vit_training.py:329-336) ----
    parser.add_argument("--data_dir", type=str, default="/datasets/imagenet-1k")
    parser.add_argument("--fake_data", action="store_true", dest="fake_data")
    parser.add_argument("--num_workers", type=int, default=4)
    parser.add_argument("--ckpt_dir", type=str, default="/tmp/vit_fsdp")
    parser.add_argument("--resume_epoch", type=int, default=0)
    parser.add_argument("--ckpt_epoch_interval", type=int, default=10)
    parser.add_argument("--test_epoch_interval", type=int, default=10)
    parser.add_argument("--log_step_interval", type=int, default=20)
    # ---- model (run_vit_training.py:339-348): defaults = ViT with 10 billion parameters ----
    parser.add_argument("--image_size", type=int, default=224)
    parser.add_argument("--patch_size", type=int, default=14)
    parser.add_argument("--embed_dim", type=int, default=5120)
    parser.add_argument("--num_heads", type=int, default=32)
    parser.add_argument("--num_blocks", type=int, default=32)
    parser.add_argument("--mlp_ratio", type=float, default=4.0)
    parser.add_argument("--pos_dropout", type=float, default=0.0)
    parser.add_argument("--att_dropout", type=float, default=0.0)
    parser.add_argument("--mlp_dropout", type=float, default=0.0)
    parser.add_argument("--num_classes", type=int, default=1000)
    # ---- optimisation (run_vit_training.py:351-361) ----
    parser.add_argument("--batch_size", type=int, default=1024)
    parser.add_argument("--num_epochs", type=int, default=300)
    parser.add_argument("--lr", type=float, default=1e-3)
    parser.add_argument("--weight_decay", type=float, default=0.1)
    parser.add_argument("--clip_grad_norm", type=float, default=1.0)
    parser.add_argument("--warmup_steps", type=int, default=10000)
    parser.add_argument("--no_grad_ckpt", action="store_false", dest="grad_ckpt")
    parser.add_argument("--no_reshard_after_forward", action="store_false", dest="reshard_after_forward")
    parser.add_argument("--flatten_parameters", action="store_true", dest="flatten_parameters")
    parser.add_argument("--run_without_fsdp", action="store_true", dest="run_without_fsdp")
    parser.add_argument("--shard_on_cpu", action="store_true", dest="shard_on_cpu")
    # ---- H100 extras (not in the reference; defaults keep reference semantics) ----
    parser.add_argument("--init_from_full_ckpt", type=str, default="",
                        help="initialise the parameters from a consolidated (unsharded) checkpoint written by "
                             "consolidate_sharded_ckpts: continues a run on a different number of GPUs "
                             "(optimizer state starts fresh; --resume_epoch restores everything but needs the same world size)")
    parser.add_argument("--ckpt_keep_blocks", type=int, default=-1,
                        help="with --grad_ckpt: how many (top) blocks keep a lean activation set instead of being "
                             "recomputed in backward; -1 = as many as the free HBM allows (measured after step 1), "
                             "0 = checkpoint every block exactly like the reference")
    parser.add_argument("--dtype", type=str, default="auto", choices=["auto", "bf16", "fp32"],
                        help="compute dtype; auto = bf16 on CUDA, fp32 on CPU")
    parser.add_argument("--backend", type=str, default="auto", choices=["auto", "sm100", "nccl", "gloo"],
                        help="collective backend: sm100 = symmetric-memory NVLink kernels, nccl/gloo = torch.distributed")
    parser.add_argument("--device", type=str, default="auto", choices=["auto", "cuda", "cpu"])
    parser.add_argument("--seed", type=int, default=0, help="parameter-init seed (identical on all ranks)")
    parser.add_argument("--init_device", type=str, default="auto", choices=["auto", "cuda", "cpu"],
                        help="where random initial parameters are drawn: auto = on the GPU for CUDA runs (fast, the "
                             "benchmarked path), on the host with --shard_on_cpu or --device cpu")
    parser.add_argument("--max_steps", type=int, default=0, help="stop every epoch after this many steps (0 = full epoch)")
    parser.add_argument("--nproc", type=int, default=0,
                        help="processes to spawn when not launched by torchrun (0 = one per visible GPU, 1 on CPU)")
    parser.add_argument("--bench_json", type=str, default="", help="append per-log-step JSON lines to this file")
    parser.add_argument("--h2d_prefetch", type=int, default=2, help="batches staged ahead on the copy stream")
    parser.add_argument("--cuda_graph", action="store_true",
                        help="capture the whole training step (fwd, bwd, collectives, clip, AdamW) in one CUDA graph")
    parser.add_argument("--drop_path_rate", type=_drop_path_rate, default=0.0,
                        help="stochastic depth (timm drop_path): block i drops each residual branch per sample with "
                             "rate linspace(0, drop_path_rate, num_blocks)[i]; 0 = off")
    # ---- batch mixing and label smoothing (timm 0.4.12 Mixup, mode 'batch'; DeiT's defaults are 0.8 / 1.0 / 0.1) ----
    parser.add_argument("--mixup", type=_non_negative("--mixup"), default=0.0,
                        help="Mixup Beta(alpha, alpha) parameter; 0 = off")
    parser.add_argument("--cutmix", type=_non_negative("--cutmix"), default=0.0,
                        help="CutMix Beta(alpha, alpha) parameter; 0 = off")
    parser.add_argument("--mixup_prob", type=_probability("--mixup_prob"), default=1.0,
                        help="probability that a step mixes its batch (when --mixup or --cutmix is on)")
    parser.add_argument("--mixup_switch_prob", type=_probability("--mixup_switch_prob"), default=0.5,
                        help="probability of CutMix instead of Mixup when both are on")
    parser.add_argument("--smoothing", type=_smoothing, default=0.0,
                        help="label smoothing of the (mixed) training targets; 0 = off")
    return parser


def _drop_path_rate(s: str) -> float:
    v = float(s)
    if not 0.0 <= v < 1.0:
        raise argparse.ArgumentTypeError(f"--drop_path_rate must be in [0, 1), got {s}")
    return v


def _non_negative(flag: str):
    def parse(s: str) -> float:
        v = float(s)
        if not (v >= 0.0 and v != float("inf")):
            raise argparse.ArgumentTypeError(f"{flag} must be a finite number >= 0, got {s}")
        return v
    return parse


def _probability(flag: str):
    def parse(s: str) -> float:
        v = float(s)
        if not 0.0 <= v <= 1.0:
            raise argparse.ArgumentTypeError(f"{flag} must be in [0, 1], got {s}")
        return v
    return parse


def _smoothing(s: str) -> float:
    v = float(s)
    if not 0.0 <= v < 1.0:
        raise argparse.ArgumentTypeError(f"--smoothing must be in [0, 1), got {s}")
    return v


def parse_args(argv=None) -> argparse.Namespace:
    return build_arg_parser().parse_args(argv)


@dataclass
class ViTConfig:
    image_size: int = 224
    patch_size: int = 14
    embed_dim: int = 5120
    num_heads: int = 32
    num_blocks: int = 32
    mlp_ratio: float = 4.0
    pos_dropout: float = 0.0
    att_dropout: float = 0.0
    mlp_dropout: float = 0.0
    num_classes: int = 1000
    drop_path_rate: float = 0.0  # stochastic depth; block i uses linspace(0, drop_path_rate, num_blocks)[i]
    mixup: float = 0.0  # Mixup / CutMix Beta alphas (0 = off), timm Mixup in 'batch' mode
    cutmix: float = 0.0
    mixup_prob: float = 1.0  # probability that a step mixes
    mixup_switch_prob: float = 0.5  # probability of CutMix when both are on
    smoothing: float = 0.0  # label smoothing of the training targets

    def __post_init__(self):
        if not 0.0 <= self.drop_path_rate < 1.0:
            raise ValueError(f"drop_path_rate must be in [0, 1), got {self.drop_path_rate}")
        for name in ("mixup", "cutmix"):
            v = getattr(self, name)
            if not (v >= 0.0 and v != float("inf")):
                raise ValueError(f"{name} must be a finite number >= 0, got {v}")
        for name in ("mixup_prob", "mixup_switch_prob"):
            if not 0.0 <= getattr(self, name) <= 1.0:
                raise ValueError(f"{name} must be in [0, 1], got {getattr(self, name)}")
        if not 0.0 <= self.smoothing < 1.0:
            raise ValueError(f"smoothing must be in [0, 1), got {self.smoothing}")

    @property
    def mixing(self) -> bool:
        """True when training steps may mix their batch (Mixup or CutMix on)."""
        return self.mixup > 0 or self.cutmix > 0

    @classmethod
    def from_args(cls, cfg) -> "ViTConfig":
        return cls(image_size=cfg.image_size, patch_size=cfg.patch_size, embed_dim=cfg.embed_dim,
                   num_heads=cfg.num_heads, num_blocks=cfg.num_blocks, mlp_ratio=cfg.mlp_ratio,
                   pos_dropout=cfg.pos_dropout, att_dropout=cfg.att_dropout, mlp_dropout=cfg.mlp_dropout,
                   num_classes=cfg.num_classes, drop_path_rate=getattr(cfg, "drop_path_rate", 0.0),
                   mixup=getattr(cfg, "mixup", 0.0), cutmix=getattr(cfg, "cutmix", 0.0),
                   mixup_prob=getattr(cfg, "mixup_prob", 1.0), mixup_switch_prob=getattr(cfg, "mixup_switch_prob", 0.5),
                   smoothing=getattr(cfg, "smoothing", 0.0))

    @property
    def grid(self) -> int:
        assert self.image_size % self.patch_size == 0, "image_size must be divisible by patch_size"
        return self.image_size // self.patch_size

    @property
    def num_patches(self) -> int:
        return self.grid * self.grid

    @property
    def head_dim(self) -> int:
        assert self.embed_dim % self.num_heads == 0
        return self.embed_dim // self.num_heads

    @property
    def hidden_dim(self) -> int:
        return int(self.embed_dim * self.mlp_ratio)

    @property
    def patch_k(self) -> int:
        return 3 * self.patch_size * self.patch_size

    @property
    def patch_kpad(self) -> int:
        """im2col K padded to a multiple of 8 elements so rows are 16-byte aligned for TMA."""
        return (self.patch_k + 7) // 8 * 8

    def block_numel(self) -> int:
        D, Hd = self.embed_dim, self.hidden_dim
        return 2 * D + (3 * D * D + 3 * D) + (D * D + D) + 2 * D + (Hd * D + Hd) + (D * Hd + D)

    def root_numel(self) -> int:
        D = self.embed_dim
        return D * self.patch_k + D + self.num_patches * D + 2 * D + self.num_classes * D + self.num_classes

    def total_numel(self) -> int:
        return self.num_blocks * self.block_numel() + self.root_numel()

    def flops_per_image(self, grad_ckpt: bool = True) -> float:
        """Matmul FLOPs of one training step per image (fwd + bwd [+ recompute])."""
        D, Hd, N = self.embed_dim, self.hidden_dim, self.num_patches
        per_block = 2 * N * (3 * D * D + D * D + 2 * D * Hd) + 4 * N * N * D
        fwd = self.num_blocks * per_block + 2 * N * self.patch_k * D + 2 * D * self.num_classes
        return fwd * (4.0 if grad_ckpt else 3.0)
