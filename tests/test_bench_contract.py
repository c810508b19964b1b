"""bench.py's command-line contract, as far as a machine without a GPU can check it: flags and defaults, the clock / throttle
sampler, the keys of the JSON line, and the reference arm's 'always one JSON line, exit 0' rule."""
import json
import os
import stat
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def test_flags_and_defaults(monkeypatch):
    import bench

    monkeypatch.setattr(sys, "argv", ["bench.py"])
    a = bench.parse()
    assert a.gpus == 1 and a.impl == "ours" and a.model == "vit10b" and a.local_batch == 128
    assert a.warmup >= 3 and 1 <= a.steps <= 20          # no flags: one GPU, finishes within minutes
    monkeypatch.setattr(sys, "argv", ["bench.py", "--gpus", "8", "--steps", "20", "--warmup", "5", "--impl", "reference"])
    a = bench.parse()
    assert (a.gpus, a.steps, a.warmup, a.impl) == (8, 20, 5, "reference")
    img, patch, dim, heads, blocks, ratio, _ = bench.MODELS["vit10b"]
    assert (img, patch, dim, heads, blocks, ratio) == (224, 14, 5120, 32, 32, 4.0)   # BASELINE.md's headline config
    assert 1 <= bench.ONE_GPU_BLOCKS < blocks and a.num_blocks == 0     # depth one 80 GB GPU holds; --num_blocks overrides
    monkeypatch.setattr(sys, "argv", ["bench.py", "--steps", "2", "--dump-outputs", "/tmp/x"])
    a = bench.parse()
    assert a.steps == 2 and a.dump_outputs == "/tmp/x"


def test_dump_outputs_writes_loss_norm_and_seeded_samples(tmp_path):
    """One CPU training step of a tiny model, then the dump: float32 arrays, same positions on every call."""
    import numpy as np
    import torch

    import bench
    from helpers import tiny_cfg
    from vit_10b_fsdp_example_b200.parallel import FSDPViT, ShardedAdamW

    cfg = tiny_cfg()
    model = FSDPViT(cfg, dtype=torch.float32, seed=0)
    opt = ShardedAdamW(model, lr=1e-3, weight_decay=0.1)
    images = torch.zeros(2, 3, cfg.image_size, cfg.image_size)
    loss = model.forward_backward(images, torch.zeros(2, dtype=torch.long))
    norm = model.clip_grad_norm_(1.0)
    opt.step()
    bench._dump_outputs(torch, model, loss, str(tmp_path / "a"), per_unit=100)
    bench._dump_outputs(torch, model, loss, str(tmp_path / "b"), per_unit=100)
    got = {n: np.load(tmp_path / "a" / f"{n}.npy") for n in ("loss", "grad_norm", "grads_sample", "weights_sample")}
    assert all(v.dtype == np.float32 for v in got.values())
    assert got["loss"][0] == np.float32(loss.item()) and got["grad_norm"][0] == np.float32(norm.item())
    n = sum(min(100, u.layout.shard_numel) for u in model.all_units)
    assert got["weights_sample"].shape == got["grads_sample"].shape == (n,)
    assert np.abs(got["grads_sample"]).max() > 0 and np.isfinite(got["weights_sample"]).all()
    for name, arr in got.items():
        assert np.array_equal(arr, np.load(tmp_path / "b" / f"{name}.npy")), name


def test_clock_sampler_parses_nvidia_smi_rows(tmp_path, monkeypatch):
    import bench

    fake = tmp_path / "nvidia-smi"
    fake.write_text("#!/bin/bash\n"
                    "echo '1305, 1965, 931.20, 0x0000000000000004, Not Active, Not Active, Not Active, Active'\n"
                    "echo '1290, 1965, 955.00, 0x0000000000000004, Not Active, Not Active, Not Active, Active'\n"
                    "echo '1335, 1965, 940.10, 0x0000000000000000, Not Active, Not Active, Not Active, Not Active'\n"
                    "echo '[N/A], broken row'\n"
                    "sleep 30\n")
    fake.chmod(fake.stat().st_mode | stat.S_IEXEC)
    monkeypatch.setenv("PATH", f"{tmp_path}:{os.environ['PATH']}")
    s = bench.ClockSampler(0)
    s.start()
    time.sleep(0.5)
    out = s.stop()
    assert out["samples"] == 3 and out["sm_mhz"] == 1305.0 and out["sm_max_mhz"] == 1965.0
    assert out["reasons"] == ["sw_power_cap"] and out["power_w_max"] == 955.0


def test_json_line_has_every_key_the_driver_reads():
    src = open(os.path.join(ROOT, "bench.py")).read()
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "model", "global_batch", "seq_len", "parallelism", "l2",
                "clocks", "sm_mhz", "sm_max_mhz", "reasons", "e2e", "h2d_bytes_per_step", "d2h_bytes_per_step",
                "gpu_launches", "impl"):
        assert f'"{key}"' in src, key
    ref = open(os.path.join(ROOT, "baseline", "reference_arm.py")).read()
    for key in ("metric", "value", "n_gpus", "ms_per_step", "e2e", "clocks", "impl", "unavailable"):
        assert f'"{key}"' in ref, key


def test_reference_arm_always_prints_one_json_line_and_exits_zero():
    """Without a GPU the reference cannot run: the arm must still exit 0 with {"impl": "reference",
    "unavailable": ...} (the rule for an arm that cannot be measured)."""
    r = subprocess.run([sys.executable, "bench.py", "--impl", "reference", "--steps", "1", "--warmup", "1"], cwd=ROOT,
                       capture_output=True, text=True, timeout=300, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    rec = json.loads(lines[0])
    assert rec["impl"] == "reference" and "unavailable" in rec
