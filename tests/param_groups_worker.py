"""Multi-process (gloo) runs of tests/dist_worker.py with optimizer parameter groups.

``opts`` takes two more keys here, ``filter_bias_and_norm`` and ``layer_decay``: every ShardedAdamW the worker builds
gets them.  Everything else (model, data, schedule, clipping, the dumped trajectory) is dist_worker's own."""
import functools
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import dist_worker  # noqa: E402


def run(rank, world, port, opts, out_path):
    from vit_10b_fsdp_example_b200 import parallel

    parallel.ShardedAdamW = functools.partial(parallel.ShardedAdamW,
                                              filter_bias_and_norm=opts.get("filter_bias_and_norm", False),
                                              layer_decay=opts.get("layer_decay"))
    dist_worker.run(rank, world, port, opts, out_path)


def launch(world, opts, out_path):
    """Every rank, W = 1 included, in a process of its own: the patched ShardedAdamW must not outlive the run."""
    import torch.multiprocessing as mp

    from helpers import free_port

    mp.spawn(run, args=(world, free_port(), opts, out_path), nprocs=world, join=True)
    with open(out_path) as f:
        return json.load(f)
