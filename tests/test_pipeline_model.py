"""Protocol model of the warp-specialised attention kernels (tools/pipeline_model.py): every kernel's mbarrier
pipeline is replayed under randomised completion orders and checked for deadlock, premature parity passes and
buffer overwrites; injected faults must be caught (so the checker is known to be sensitive)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pipeline_model as pm  # noqa: E402

SEEDS = range(40)


@pytest.mark.parametrize("nt", [1, 2, 3, 4, 9])
@pytest.mark.parametrize("ts_bufs,kT", [(2, True), (1, True), (2, False)])
def test_one_shot_backward_protocol(nt, ts_bufs, kT):
    """attention_bwd_sm100.cu (validated on hardware): also calibrates the model."""
    for seed in SEEDS:
        pm.model_bwd(seed, 1, nt, ts_bufs, 4, kT, persistent=False)


@pytest.mark.parametrize("n_items,nt", [(1, 4), (2, 1), (3, 3), (4, 4), (2, 9)])
@pytest.mark.parametrize("kT", [True, False])
def test_persistent_backward_protocol(n_items, nt, kT):
    for seed in SEEDS:
        pm.model_bwd(seed, n_items, nt, 2, 8, kT, persistent=True)


@pytest.mark.parametrize("n_items,nkt", [(1, 4), (3, 4), (4, 3), (5, 1), (3, 2)])
def test_persistent_forward_protocol(n_items, nkt):
    for seed in SEEDS:
        pm.model_fwd_persist(seed, n_items, nkt)


@pytest.mark.parametrize("nt", [1, 2, 5, 9, 16])
def test_long_forward_protocol(nt):
    for seed in SEEDS:
        pm.model_fwd_long(seed, nt)


@pytest.mark.parametrize("bug,args", [
    ("no_x_empty", dict(n_items=3, nt=4, ts_bufs=2, warps=8, kT=True, persistent=True)),
    ("y_empty_parity", dict(n_items=3, nt=4, ts_bufs=2, warps=8, kT=True, persistent=True)),
    ("no_e_empty", dict(n_items=1, nt=4, ts_bufs=2, warps=4, kT=True, persistent=False)),
    ("no_ts_empty", dict(n_items=1, nt=4, ts_bufs=1, warps=4, kT=True, persistent=False)),  # single T_s buffer
])
def test_injected_faults_are_detected(bug, args):
    caught = 0
    for seed in range(60):
        try:
            pm.model_bwd(seed, bug=bug, **args)
        except pm.ProtocolError:
            caught += 1
    assert caught > 0, f"fault {bug} was never detected"


def test_forward_softmax_to_epilogue_handoff_needs_its_mbarrier():
    """Round-2 forward: 1 / row sum travels from the softmax warps to the separate epilogue warps through a plain
    shared-memory slot ordered only by the stat_full mbarrier (the pair compute-sanitizer racecheck flags, see
    of the kernel tests).  With the wait the protocol holds for every schedule; without it the model must see
    the epilogue read a slot that is stale or half written."""
    for seed in range(120):
        pm.model_fwd_persist(seed, 5, 4)
    caught = 0
    for seed in range(60):
        try:
            pm.model_fwd_persist(seed, 5, 4, bug="no_stat_full")
        except pm.ProtocolError:
            caught += 1
    assert caught == 60


def test_statistics_stage_of_the_persistent_backward():
    """Round-2 dK/dV role: per-query statistics arrive as bulk copies into a 2-stage buffer.  The model holds with the
    stat_empty wait and -- like acc_empty -- also without it: a stage is only re-requested after x_empty of the next
    item, which every softmax warp can only enable after it has left the previous item (belt-and-braces wait)."""
    for seed in range(60):
        pm.model_bwd(seed, 5, 3, 2, 8, True, persistent=True)
        pm.model_bwd(seed, 5, 1, 2, 8, True, persistent=True, bug="no_stat_empty")


@pytest.mark.parametrize("tiles,clusters,num_kb,stages,epi_warps", [
    (7, 2, 3, 3, 8),     # the kernel's shape: 8 epilogue warps per CTA, 20 consumers per CLC response
    (5, 3, 2, 2, 2),
    (1, 1, 1, 3, 2),     # a single tile: no CLC response is ever a valid tile
    (2, 3, 5, 2, 2),     # more resident clusters than tiles
    (12, 2, 1, 2, 2),    # short K (attention GEMMs): the epilogue, not the MMA, sets the pace
])
def test_gemm_cta_pair_clc_protocol(tiles, clusters, num_kb, stages, epi_warps):
    """gemm_sm100.cu: TMA producers of both CTAs signalling the leader's barrier, multicast commits, double-buffered
    TMEM accumulator, cluster-launch-control work stealing with multicast responses."""
    for seed in range(25):
        pm.model_gemm(seed, tiles, clusters, num_kb, stages, epi_warps=epi_warps, epi_delay=40)
        pm.model_gemm(seed, tiles, clusters, num_kb, stages, epi_warps=epi_warps, use_clc=False)  # static persistent grid


@pytest.mark.parametrize("bug", ["no_empty", "no_tmem_empty", "no_clc_empty", "peer_arms_too"])
def test_gemm_injected_faults_are_detected(bug):
    caught = 0
    for seed in range(40):
        try:
            pm.model_gemm(seed, 9, clusters=2, num_kb=1 if bug == "no_tmem_empty" else 3, stages=2, epi_warps=2,
                          epi_delay=200, bug=bug)
        except pm.ProtocolError:
            caught += 1
    assert caught > 0, f"fault {bug} was never detected"
