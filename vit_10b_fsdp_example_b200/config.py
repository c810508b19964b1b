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
    parser.add_argument("--qk_norm", action="store_true",
                        help="QK normalisation (timm Attention(qk_norm=True), ViT-22B): a LayerNorm over the head dim "
                             "of every query and key head before the attention scores, with learned weight and bias "
                             "per block; keeps the attention logits bounded at large scale")
    parser.add_argument("--init_values", type=_non_negative("--init_values"), default=0.0,
                        help="LayerScale (CaiT, timm VisionTransformer(init_values=...)): every block scales its "
                             "attention and MLP branches by learned per-channel vectors ls1.gamma / ls2.gamma that "
                             "start at this value (1e-5 to 1e-4 in DeiT III / DINOv2 recipes); 0 = off")
    # ---- prefix tokens (timm VisionTransformer(class_token=..., reg_tokens=..., no_embed_class=...)) ----
    parser.add_argument("--class_token", action="store_true",
                        help="prepend a learned class token (cls_token) to every image's patch tokens and classify "
                             "from it after the final norm (timm global_pool='token'; DeiT, DeiT III, DINOv2) instead "
                             "of mean-pooling the patches")
    parser.add_argument("--reg_tokens", type=_reg_tokens, default=0,
                        help="learned register tokens placed after the class token (Darcet et al., 2023, 'Vision "
                             "Transformers Need Registers'); needs --class_token; 0 = none")
    parser.add_argument("--no_embed_class", action="store_true",
                        help="pos_embed covers the patches only and the class / register tokens get no position "
                             "embedding (timm no_embed_class=True); needs --class_token")
    parser.add_argument("--swiglu", action="store_true",
                        help="SwiGLU MLP (timm mlp_layer=SwiGLUPacked, act_layer=nn.SiLU; Shazeer 2020, DINOv2-g): "
                             "fc1 makes Hd = int(embed_dim * mlp_ratio) features [gate | value], fc2 reads "
                             "silu(gate) * value of width Hd / 2; Hd must be a multiple of 16")
    parser.add_argument("--patch_drop_rate", type=_patch_drop_rate, default=0.0,
                        help="patch dropout (timm PatchDropout; Liu et al. 2022, FLIP): in training every image keeps "
                             "a random max(1, int(N * (1 - rate))) of its N patch tokens (the class / register tokens "
                             "always), so every block runs on fewer tokens; evaluation keeps all; 0 = off")
    # ---- rotary position embedding (EVA-02: timm Eva(use_rot_pos_emb=True), RotaryEmbeddingCat) ----
    parser.add_argument("--rope", action="store_true",
                        help="2-D axial rotary position embedding (EVA-02, timm RotaryEmbeddingCat) on the queries and "
                             "keys of every block, after --qk_norm, on top of the learned pos_embed: of the hd / 2 "
                             "interleaved pairs of a head, the first hd / 4 turn with the patch row, the rest with the "
                             "patch column; class and register tokens are not rotated; needs head_dim % 4 == 0")
    parser.add_argument("--rope_theta", type=_rope_theta, default=ROPE_THETA,
                        help="RoPE base theta: pair j of a half turns with frequency theta ** (-j / (head_dim / 4)); "
                             "needs --rope")
    parser.add_argument("--rope_ref_grid", type=_rope_ref_grid, default=0,
                        help="RoPE reference grid g_ref (timm ref_feat_shape): positions are scaled by g_ref / grid, "
                             "so a fine-tune at a higher resolution keeps the pre-training angles when g_ref is the "
                             "pre-training grid; 0 = the run's own grid; needs --rope")
    # ---- model EMA (timm ModelEmaV2; DeiT --model-ema) ----
    parser.add_argument("--model_ema", action="store_true",
                        help="keep an exponential moving average of the weights (timm ModelEmaV2, DeiT --model-ema), "
                             "sharded like the master and updated by every optimizer step; it starts as a copy of the "
                             "initial (or --init_from_full_ckpt) weights, is evaluated after the model at every test "
                             "epoch and is saved as model_ema in the checkpoints; 4 bytes per sharded parameter")
    parser.add_argument("--model_ema_decay", type=_ema_decay, default=0.9998,
                        help="EMA decay d: ema = d * ema + (1 - d) * w after every step (timm train.py 0.9998, DeiT "
                             "0.99996); in [0, 1), 0 = the EMA is the weights")
    # ---- optimizer parameter groups (MAE param_groups_lrd; timm create_optimizer_v2 filter_bias_and_bn / --layer-decay) ----
    parser.add_argument("--filter_bias_and_norm", action="store_true",
                        help="no weight decay on parameters that are 1-D in timm's layout (biases, LayerNorm and q/k "
                             "norm weights, LayerScale gammas) nor on pos_embed, cls_token and reg_token (timm "
                             "filter_bias_and_bn, DeiT, MAE); off = decay every tensor like the reference")
    parser.add_argument("--layer_decay", type=_layer_decay, default=None,
                        help="layer-wise lr decay d (BEiT / MAE / DINOv2 fine-tuning, timm --layer-decay): block i trains "
                             "at lr * d ** (num_blocks - i), the stem (patch_embed, pos_embed, tokens) at "
                             "lr * d ** (num_blocks + 1), the final norm and head at lr; in (0, 1], typically 0.65-0.75; "
                             "implies --filter_bias_and_norm (1 = the filter alone)")
    return parser


def check_swiglu(cfg) -> None:
    """The SwiGLU value half starts at column Hd / 2 of the packed fc1 output: the GEMM's second store map and the
    16-byte vectors of the SwiGLU kernels need that column 16-byte aligned, so Hd % 16 == 0 (timm only needs Hd even)."""
    if getattr(cfg, "swiglu", False):
        hd = int(cfg.embed_dim * cfg.mlp_ratio)
        if hd % 16 != 0:
            raise ValueError(f"--swiglu needs the MLP width Hd = int(embed_dim * mlp_ratio) to be a multiple of 16 "
                             f"(the value half starts at column Hd / 2, which must be 16-byte aligned); got Hd = {hd}")


def check_prefix_flags(args) -> None:
    """--reg_tokens and --no_embed_class only mean something next to a class token."""
    if not args.class_token and (args.reg_tokens or args.no_embed_class):
        flag = "--reg_tokens" if args.reg_tokens else "--no_embed_class"
        raise ValueError(f"{flag} needs --class_token (register tokens and an un-embedded prefix exist only next to a "
                         f"class token; mean pooling has no prefix tokens)")


ROPE_THETA = 10000.0  # timm RotaryEmbeddingCat temperature


def check_rope(cfg) -> None:
    """--rope_theta / --rope_ref_grid only mean something with --rope, and the rotation splits every head into two
    halves of interleaved pairs, so --rope needs head_dim % 4 == 0."""
    rope = getattr(cfg, "rope", False)
    if not rope and (getattr(cfg, "rope_theta", ROPE_THETA) != ROPE_THETA or getattr(cfg, "rope_ref_grid", 0)):
        flag = "--rope_theta" if getattr(cfg, "rope_theta", ROPE_THETA) != ROPE_THETA else "--rope_ref_grid"
        raise ValueError(f"{flag} needs --rope (it sets the rotary position embedding, which is off)")
    if rope and cfg.embed_dim % cfg.num_heads == 0 and (cfg.embed_dim // cfg.num_heads) % 4 != 0:
        raise ValueError(f"--rope needs head_dim % 4 == 0 (hd / 4 frequency pairs for the patch row and as many for the "
                         f"column), got head_dim = {cfg.embed_dim // cfg.num_heads}")


def _rope_theta(s: str) -> float:
    v = float(s)
    if not (v > 0.0 and v != float("inf")):
        raise argparse.ArgumentTypeError(f"--rope_theta must be a finite number > 0, got {s}")
    return v


def _rope_ref_grid(s: str) -> int:
    v = int(s)
    if v < 0:
        raise argparse.ArgumentTypeError(f"--rope_ref_grid must be an integer >= 0, got {s}")
    return v


def _drop_path_rate(s: str) -> float:
    v = float(s)
    if not 0.0 <= v < 1.0:
        raise argparse.ArgumentTypeError(f"--drop_path_rate must be in [0, 1), got {s}")
    return v


def _patch_drop_rate(s: str) -> float:
    v = float(s)
    if not 0.0 <= v < 1.0:
        raise argparse.ArgumentTypeError(f"--patch_drop_rate must be in [0, 1), got {s}")
    return v


def _ema_decay(s: str) -> float:
    v = float(s)
    if not 0.0 <= v < 1.0:
        raise argparse.ArgumentTypeError(f"--model_ema_decay must be in [0, 1), got {s}")
    return v


def _layer_decay(s: str) -> float:
    v = float(s)
    if not 0.0 < v <= 1.0:
        raise argparse.ArgumentTypeError(f"--layer_decay must be in (0, 1], got {s}")
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


def _reg_tokens(s: str) -> int:
    v = int(s)
    if v < 0:
        raise argparse.ArgumentTypeError(f"--reg_tokens must be an integer >= 0, got {s}")
    return v


def _smoothing(s: str) -> float:
    v = float(s)
    if not 0.0 <= v < 1.0:
        raise argparse.ArgumentTypeError(f"--smoothing must be in [0, 1), got {s}")
    return v


def parse_args(argv=None) -> argparse.Namespace:
    parser = build_arg_parser()
    args = parser.parse_args(argv)
    try:
        check_prefix_flags(args)
        check_swiglu(args)
        check_rope(args)
    except ValueError as e:
        parser.error(str(e))
    return args


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
    qk_norm: bool = False  # per-head LayerNorm on q and k (timm Attention(qk_norm=True))
    init_values: float = 0.0  # LayerScale initial value (timm VisionTransformer(init_values=...)); 0 = off
    class_token: bool = False  # learned cls_token in front of the patches, classified from (timm global_pool='token')
    reg_tokens: int = 0  # learned register tokens after the class token (needs class_token)
    no_embed_class: bool = False  # pos_embed covers the patches only (timm no_embed_class=True; needs class_token)
    swiglu: bool = False  # SwiGLU MLP (timm SwiGLUPacked): fc1 -> [gate | value] of width hidden_dim, fc2 reads half of it
    patch_drop_rate: float = 0.0  # patch dropout in training (timm PatchDropout, ordered); 0 = off
    rope: bool = False  # 2-D axial rotary position embedding on q and k (EVA-02, timm RotaryEmbeddingCat)
    rope_theta: float = ROPE_THETA  # RoPE base
    rope_ref_grid: int = 0  # RoPE reference grid (timm ref_feat_shape); 0 = the run's grid

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
        if not (self.init_values >= 0.0 and self.init_values != float("inf")):
            raise ValueError(f"init_values must be a finite number >= 0, got {self.init_values}")
        if not (isinstance(self.reg_tokens, int) and self.reg_tokens >= 0):
            raise ValueError(f"reg_tokens must be an integer >= 0, got {self.reg_tokens}")
        if not 0.0 <= self.patch_drop_rate < 1.0:
            raise ValueError(f"patch_drop_rate must be in [0, 1), got {self.patch_drop_rate}")
        if not (self.rope_theta > 0.0 and self.rope_theta != float("inf")):
            raise ValueError(f"rope_theta must be a finite number > 0, got {self.rope_theta}")
        if not (isinstance(self.rope_ref_grid, int) and self.rope_ref_grid >= 0):
            raise ValueError(f"rope_ref_grid must be an integer >= 0, got {self.rope_ref_grid}")
        check_prefix_flags(self)
        check_swiglu(self)
        check_rope(self)

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
                   smoothing=getattr(cfg, "smoothing", 0.0), qk_norm=getattr(cfg, "qk_norm", False),
                   init_values=getattr(cfg, "init_values", 0.0), class_token=getattr(cfg, "class_token", False),
                   reg_tokens=getattr(cfg, "reg_tokens", 0), no_embed_class=getattr(cfg, "no_embed_class", False),
                   swiglu=getattr(cfg, "swiglu", False), patch_drop_rate=getattr(cfg, "patch_drop_rate", 0.0),
                   rope=getattr(cfg, "rope", False), rope_theta=getattr(cfg, "rope_theta", ROPE_THETA),
                   rope_ref_grid=getattr(cfg, "rope_ref_grid", 0))

    @property
    def grid(self) -> int:
        assert self.image_size % self.patch_size == 0, "image_size must be divisible by patch_size"
        return self.image_size // self.patch_size

    @property
    def num_patches(self) -> int:
        return self.grid * self.grid

    @property
    def num_prefix_tokens(self) -> int:
        """P: the class token and the register tokens in front of every image's patches (0 without a class token)."""
        return (1 + self.reg_tokens) if self.class_token else 0

    @property
    def num_tokens(self) -> int:
        """T = N + P: the tokens per image every block runs on."""
        return self.num_patches + self.num_prefix_tokens

    @property
    def num_keep(self) -> int:
        """K: the patches every image keeps in a training step, max(1, int(N * (1 - patch_drop_rate))) in float64 as
        timm's PatchDropout computes it (N at rate 0)."""
        return max(1, int(self.num_patches * (1.0 - float(self.patch_drop_rate))))

    @property
    def train_tokens(self) -> int:
        """T' = P + K: the tokens per image every block runs on in a training step (num_tokens at rate 0)."""
        return self.num_prefix_tokens + self.num_keep

    @property
    def pos_len(self) -> int:
        """Rows of pos_embed: every token, or only the patches under no_embed_class."""
        return self.num_patches if self.no_embed_class else self.num_tokens

    @property
    def head_dim(self) -> int:
        assert self.embed_dim % self.num_heads == 0
        return self.embed_dim // self.num_heads

    @property
    def hidden_dim(self) -> int:
        return int(self.embed_dim * self.mlp_ratio)

    @property
    def mlp_out_dim(self) -> int:
        """Width of the fc2 input: hidden_dim, or with SwiGLU the hidden_dim / 2 columns of silu(gate) * value."""
        return self.hidden_dim // 2 if self.swiglu else self.hidden_dim

    @property
    def patch_k(self) -> int:
        return 3 * self.patch_size * self.patch_size

    @property
    def patch_kpad(self) -> int:
        """im2col K padded to a multiple of 8 elements so rows are 16-byte aligned for TMA."""
        return (self.patch_k + 7) // 8 * 8

    def block_numel(self) -> int:
        D, Hd = self.embed_dim, self.hidden_dim
        qk = 4 * self.head_dim if self.qk_norm else 0  # q_norm / k_norm weight and bias
        ls = 2 * D if self.init_values else 0  # ls1.gamma / ls2.gamma
        return 2 * D + (3 * D * D + 3 * D) + qk + (D * D + D) + 2 * D + (Hd * D + Hd) + (D * self.mlp_out_dim + D) + ls

    def root_numel(self) -> int:
        D = self.embed_dim
        return (D * self.patch_k + D + self.num_prefix_tokens * D + self.pos_len * D + 2 * D + self.num_classes * D
                + self.num_classes)

    def total_numel(self) -> int:
        return self.num_blocks * self.block_numel() + self.root_numel()

    def flops_per_image(self, grad_ckpt: bool = True) -> float:
        """Matmul FLOPs of one training step per image (fwd + bwd [+ recompute])."""
        D, Hd, N, T = self.embed_dim, self.hidden_dim, self.num_patches, self.num_tokens
        per_block = 2 * T * (3 * D * D + D * D + D * Hd + D * self.mlp_out_dim) + 4 * T * T * D
        fwd = self.num_blocks * per_block + 2 * N * self.patch_k * D + 2 * D * self.num_classes
        return fwd * (4.0 if grad_ckpt else 3.0)
