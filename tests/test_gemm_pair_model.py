"""Protocol model of the H100 GEMM's 2-CTA clusters (tools/pipeline_model.py, model_gemm_sm90_pair): the multicast
B tile, the 16-arrival empty barriers and the teardown cluster sync replayed under randomised schedules; injected
faults must be caught, so the checker is known to see them."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pipeline_model as pm  # noqa: E402


@pytest.mark.parametrize("m_tiles,n_tiles,batch,clusters,num_kb,stages", [
    (2, 3, 1, 2, 3, 3),   # one pair per column, several units per cluster
    (5, 2, 1, 2, 4, 4),   # odd m-tile count: the last pair's second CTA is below the matrix
    (1, 3, 2, 2, 2, 3),   # a single m-tile per batch entry
    (3, 2, 2, 3, 3, 2),   # odd per batch entry, batched, more k-blocks than stages
    (4, 4, 1, 1, 5, 4),   # one cluster walks every unit
    (2, 1, 1, 3, 2, 2),   # more clusters than units: idle clusters still meet their syncs
])
def test_gemm_pair_protocol(m_tiles, n_tiles, batch, clusters, num_kb, stages):
    for seed in range(40):
        pm.model_gemm_sm90_pair(seed, m_tiles, n_tiles, batch, clusters, num_kb, stages)


@pytest.mark.parametrize("bug", ["local_only", "no_final_sync", "wait_peer_full"])
def test_gemm_pair_injected_faults_are_detected(bug):
    caught = 0
    for seed in range(60):
        try:
            pm.model_gemm_sm90_pair(seed, 3, 2, batch=2, clusters=2, num_kb=3, stages=2, bug=bug)
        except pm.ProtocolError:
            caught += 1
    assert caught > 0, f"fault {bug} was never detected"
