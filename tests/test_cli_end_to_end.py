"""The flag-compatible entry point end to end on CPU/gloo (BASELINE.md's plumbing config: ViT-Tiny-like, W=2, --fake_data):
train -> per-rank checkpoints -> resume -> evaluate -> offline consolidation, all through the command line."""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = ["--fake_data", "--device", "cpu", "--nproc", "2", "--image_size", "32", "--patch_size", "8", "--embed_dim", "32",
        "--num_heads", "2", "--num_blocks", "2", "--num_classes", "10", "--batch_size", "8", "--warmup_steps", "2",
        "--lr", "1e-2", "--max_steps", "3", "--log_step_interval", "1", "--num_workers", "0",
        "--ckpt_epoch_interval", "1", "--test_epoch_interval", "1", "--ckpt_keep_blocks", "1"]


def _run(args, timeout=300):
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    return subprocess.run([sys.executable] + args, cwd=ROOT, env=env, capture_output=True, text=True, timeout=timeout)


def test_train_resume_consolidate_via_cli(tmp_path):
    ckpt = str(tmp_path / "ckpt")
    jsonl = str(tmp_path / "steps.jsonl")
    r = _run(["run_vit_training.py", *TINY, "--ckpt_dir", ckpt, "--num_epochs", "1", "--bench_json", jsonl])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = r.stdout
    assert "training completed" in out and "accuracy on val" in out
    import json
    rows = [json.loads(line) for line in open(jsonl)]  # --bench_json: one JSON line per logged step, rank 0 only
    assert [row["step"] for row in rows] == [1, 2, 3] and all(row["images_per_sec"] > 0 for row in rows)
    assert rows[0]["lr"] == 0.005 and rows[-1]["loss"] < rows[0]["loss"]
    assert "epoch 1 step 1, lr:" in out and "sec/iter" in out  # the reference's log line
    for rank in (0, 1):
        assert os.path.exists(os.path.join(ckpt, f"epoch_1_rank_{rank}.ckpt"))
    state = torch.load(os.path.join(ckpt, "epoch_1_rank_0.ckpt"), map_location="cpu", weights_only=False)
    assert set(state) == {"model", "shard_metadata", "optimizer", "lr_scheduler"}

    # resume from epoch 1 and train epoch 2 (all-zero images with label 0: the loss keeps falling)
    r2 = _run(["run_vit_training.py", *TINY, "--ckpt_dir", ckpt, "--num_epochs", "2", "--resume_epoch", "1"])
    assert r2.returncode == 0, r2.stdout[-2000:] + r2.stderr[-2000:]
    assert "starting epoch 2" in r2.stdout and "starting epoch 1" not in r2.stdout
    assert os.path.exists(os.path.join(ckpt, "epoch_2_rank_1.ckpt"))

    # offline consolidation of the two rank files into one unsharded state_dict with timm-style names / shapes
    full = str(tmp_path / "full.pth")
    r3 = _run(["-m", "vit_10b_fsdp_example_b200.consolidate_sharded_ckpts", "--ckpt_prefix",
               os.path.join(ckpt, "epoch_2"), "--save_path", full])
    assert r3.returncode == 0, r3.stdout[-2000:] + r3.stderr[-2000:]
    sd = torch.load(full, map_location="cpu", weights_only=False)
    sd = sd.get("model", sd)
    assert sd["blocks.0.attn.qkv.weight"].shape == (96, 32)
    assert sd["pos_embed"].shape == (1, 16, 32) and sd["head.weight"].shape == (10, 32)

    # continue on ONE process from the consolidated file (different world size than the run that wrote the shards)
    one = [a if a != "2" or TINY[i - 1] != "--nproc" else "1" for i, a in enumerate(TINY)]
    r4 = _run(["run_vit_training.py", *one, "--ckpt_dir", str(tmp_path / "ckpt1"), "--num_epochs", "1",
               "--init_from_full_ckpt", full])
    assert r4.returncode == 0, r4.stdout[-2000:] + r4.stderr[-2000:]
    assert "parameters initialised from the consolidated checkpoint" in r4.stdout and "training completed" in r4.stdout


def test_pod_launch_runs_two_nodes_through_a_local_transport(tmp_path):
    """The multi-host launcher for real (not --dry-run): two 'hosts' reached through a stand-in for ssh that runs the
    per-host command locally, one process per node, 2-node torchrun rendezvous on 127.0.0.1, the training CLI on
    gloo.  Role of the xla_dist pod launch in the reference (README.md:99-118)."""
    import socket

    fake_ssh = tmp_path / "local_ssh.sh"
    fake_ssh.write_text('#!/bin/bash\n# usage: local_ssh.sh <host> <command>: run the command here\nshift\nexec bash -c "$1"\n')
    fake_ssh.chmod(0o755)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    tiny = [a for i, a in enumerate(TINY) if a != "--nproc" and TINY[i - 1] != "--nproc"]
    ckpt = str(tmp_path / "ckpt")
    r = _run(["-m", "vit_10b_fsdp_example_b200.pod_launch", "--hosts", "127.0.0.1,127.0.0.1", "--nproc-per-node", "1",
              "--master-port", str(port), "--ssh", str(fake_ssh), "--workdir", ROOT, "--python", sys.executable,
              "--env", "OMP_NUM_THREADS=1", "--env", "POD_LAUNCH_TEST=forwarded value",
              "--", "run_vit_training.py", *tiny, "--ckpt_dir", ckpt, "--num_epochs", "1"], timeout=420)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "training completed" in r.stdout
    for rank in (0, 1):  # one rank per node, both wrote their shard
        assert os.path.exists(os.path.join(ckpt, f"epoch_1_rank_{rank}.ckpt"))

    # a failing host takes the job down with a non-zero exit code
    bad = _run(["-m", "vit_10b_fsdp_example_b200.pod_launch", "--hosts", "127.0.0.1", "--nproc-per-node", "1",
                "--master-port", str(port), "--ssh", str(fake_ssh), "--workdir", ROOT, "--python", sys.executable,
                "--", "run_vit_training.py", "--no_such_flag"], timeout=120)
    assert bad.returncode != 0


def test_real_image_folder_through_the_cli(tmp_path):
    """Not --fake_data: a generated ImageFolder tree, the reference's transforms, DataLoader workers, DistributedSampler
    (set_epoch), two ranks, two epochs, evaluation on the val split (reference run_vit_training.py:39-88,283-302)."""
    from PIL import Image

    g = torch.Generator().manual_seed(0)
    for split, per_class in (("train", 16), ("val", 8)):
        for c, cls in enumerate(("n01", "n02")):
            d = tmp_path / "data" / split / cls
            d.mkdir(parents=True)
            for i in range(per_class):
                arr = (torch.rand(40, 48, 3, generator=g) * 80 + 160 * c).to(torch.uint8).numpy()  # dark vs bright
                Image.fromarray(arr).save(d / f"img_{i}.jpeg")
    args = [a for i, a in enumerate(TINY) if a not in ("--fake_data", "--max_steps", "--num_workers")
            and TINY[i - 1] not in ("--max_steps", "--num_workers")]
    ckpt = str(tmp_path / "ckpt")
    r = _run(["run_vit_training.py", *args, "--data_dir", str(tmp_path / "data"), "--num_workers", "2", "--num_classes", "2",
              "--ckpt_dir", ckpt, "--num_epochs", "2"])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = r.stdout
    assert "loading images from directory" in out and "training completed" in out
    assert "epoch 2 step 4" in out  # 32 train images / global batch 8 = 4 steps per epoch
    assert out.count("accuracy on val") == 2
    assert os.path.exists(os.path.join(ckpt, "epoch_2_rank_1.ckpt"))


def test_every_strategy_flag_through_the_cli_gives_the_same_trajectory(tmp_path):
    """The reference's strategy flags (run_vit_training.py:323-331) reach the engine through the command line: ZeRO-3
    default, ZeRO-2-like, flattened, no activation checkpointing, host-side sharded init, plain DDP and dropout-free
    single process all print the same loss trajectory (same seed, all-zero images, label 0)."""
    import re

    base = [a for i, a in enumerate(TINY) if a not in ("--ckpt_keep_blocks", "--nproc")
            and TINY[i - 1] not in ("--ckpt_keep_blocks", "--nproc")]
    variants = {
        "zero3": ["--nproc", "2"],
        "zero2_flat": ["--nproc", "2", "--no_reshard_after_forward", "--flatten_parameters"],
        "no_ckpt_cpu_init": ["--nproc", "2", "--no_grad_ckpt", "--shard_on_cpu"],
        "ddp": ["--nproc", "2", "--run_without_fsdp"],
        "keep_all": ["--nproc", "2", "--ckpt_keep_blocks", "2"],
        "single": ["--nproc", "1"],
    }
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    procs = {name: subprocess.Popen([sys.executable, "run_vit_training.py", *base, *extra, "--ckpt_dir",
                                     str(tmp_path / name), "--num_epochs", "1"], cwd=ROOT, env=env,
                                    stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for name, extra in variants.items()}  # the six jobs are independent: run them side by side
    losses = {}
    for name, proc in procs.items():
        out, err = proc.communicate(timeout=600)
        assert proc.returncode == 0, name + out[-2000:] + err[-2000:]
        losses[name] = [float(x) for x in re.findall(r"loss: ([0-9.]+)", out)]
        assert len(losses[name]) == 3, (name, out[-1500:])
    ref = losses["zero3"]
    assert ref[2] < ref[0]
    for name, ls in losses.items():
        for a, b in zip(ls, ref):
            assert abs(a - b) < 2e-3, (name, ls, ref)


def test_a_dying_rank_takes_the_job_down_and_resume_continues(tmp_path):
    """Failure contract: a rank that crashes mid-epoch must not leave its peers hanging in a collective --
    the launcher exits non-zero in bounded time -- and the run continues from the last checkpoint with --resume_epoch."""
    ckpt = str(tmp_path / "ckpt")
    ok = _run(["run_vit_training.py", *TINY, "--ckpt_dir", ckpt, "--num_epochs", "1"])
    assert ok.returncode == 0, ok.stdout[-2000:] + ok.stderr[-2000:]
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1", B200_INJECT_FAILURE="1:2:2")
    bad = subprocess.run([sys.executable, "run_vit_training.py", *TINY, "--ckpt_dir", ckpt, "--num_epochs", "3",
                          "--resume_epoch", "1"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=120)
    assert bad.returncode != 0
    assert "[fault injection] rank 1 dies at epoch 2 step 2" in bad.stdout
    assert "training completed" not in bad.stdout
    assert not os.path.exists(os.path.join(ckpt, "epoch_2_rank_0.ckpt"))  # nothing half-written was left behind
    again = _run(["run_vit_training.py", *TINY, "--ckpt_dir", ckpt, "--num_epochs", "3", "--resume_epoch", "1"])
    assert again.returncode == 0, again.stdout[-2000:] + again.stderr[-2000:]
    assert "starting epoch 2" in again.stdout and "training completed" in again.stdout
    assert os.path.exists(os.path.join(ckpt, "epoch_3_rank_1.ckpt"))
