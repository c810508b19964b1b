#!/usr/bin/env python
"""ViT-10B FSDP training on H100 -- flag-compatible entry point.

Accepts the reference's command line unchanged (run_vit_training.py:327-363), e.g.

    python run_vit_training.py --fake_data --batch_size 1024 --shard_on_cpu
    torchrun --standalone --nproc-per-node 8 run_vit_training.py --fake_data

Without torchrun it spawns one process per visible GPU (the role xmp.spawn plays in the reference).
"""
from vit_10b_fsdp_example_b200.config import parse_args
from vit_10b_fsdp_example_b200.launch import launch
from vit_10b_fsdp_example_b200.train import main

if __name__ == "__main__":
    cfg = parse_args()
    launch(main, cfg)
