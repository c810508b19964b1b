"""Equivalence matrix: every sharding / scheduling flag must leave the numerics unchanged.

FSDP (W=1,2,4) x --run_without_fsdp x grad-ckpt x reshard x flatten x shard_on_cpu all have to produce the
same loss / grad-norm trajectory as the single-process run on the same global batch.
"""
import pytest

from dist_worker import launch


def _close(a, b, tol=2e-5):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert abs(x - y) <= tol * max(1.0, abs(y)), (a, b)


@pytest.fixture(scope="module")
def baseline(tmp_path_factory):
    out = tmp_path_factory.mktemp("base") / "r.json"
    return launch(1, {"steps": 4}, str(out))


@pytest.mark.parametrize("world,opts", [
    (2, {}),
    (2, {"flatten": True}),
    (2, {"reshard": False}),
    (2, {"grad_ckpt": False}),
    (2, {"keep_blocks": 1}),
    (2, {"poison": True}),
    (2, {"poison": True, "grad_ckpt": False, "reshard": False}),
    (2, {"shard_on_cpu": True, "flatten": True, "grad_ckpt": False, "reshard": False}),
    (2, {"no_fsdp": True}),
    (4, {}),
    (8, {}),                                   # the flagship world size: one image per rank, 8-way shards with padding
    (8, {"flatten": True, "reshard": False}),
    (1, {"flatten": True, "grad_ckpt": False}),
    (1, {"no_fsdp": True}),
])
def test_same_trajectory(world, opts, baseline, tmp_path):
    res = launch(world, dict(opts, steps=4), str(tmp_path / "r.json"))
    _close(res["losses"], baseline["losses"])
    _close(res["norms"], baseline["norms"], tol=1e-4)


def test_sharded_param_count(tmp_path):
    r1 = launch(1, {"steps": 1}, str(tmp_path / "a.json"))
    r2 = launch(2, {"steps": 1}, str(tmp_path / "b.json"))
    # ZeRO-3: a rank owns ~1/W of the parameters (up to alignment padding)
    assert r2["sharded"] < 0.55 * r1["sharded"]
