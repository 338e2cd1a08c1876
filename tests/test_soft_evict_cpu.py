"""Preempt with PreferNoSchedule taints on the CPU oracles: the hand-derived sessions of tests/soft_cases.py give the
derived statements through the unchanged oracle (oracle/oracle.cpp, no sampling) and through the sampling oracle
(tools/samp_evict_oracle, every case); the topology-aware reading (tools/topo_oracle) does not score nodes, so its
statements do not depend on tainttoleration.weight. The device path is measured against these oracles."""
import pytest

from tests import samp_cases as SC
from tests import samp_common as S
from tests import soft_cases as SOFT
from volcano_b200.snapshot import PreemptArguments


@pytest.mark.parametrize("case", sorted(SOFT.CASES))
def test_sampling_oracle_gives_the_derived_statements(case):
    snap, want = SOFT.CASES[case]()
    res = S.run(snap)
    assert SC.statements(snap, res.preempt) == want


@pytest.mark.parametrize("case", ["all_nodes", "zero_max"])
def test_unchanged_oracle_gives_the_derived_statements(case):
    snap, want = SOFT.CASES[case]()
    res = S.run(snap, restated=False)
    assert SC.statements(snap, res.preempt) == want


def test_topology_aware_reading_ignores_the_taint_score():
    """all_nodes_case in the topology-aware reading, numCandidates large enough for every candidate to compete: the
    statements are the same at tainttoleration.weight 3 and 0 (pickOneNodeForPreemption's four criteria,
    preempt.go:850-1015, read victims and start times only)."""
    out = []
    for weight in (3, 0):
        SOFT.NODEORDER_ARGS["tainttoleration.weight"] = weight
        try:
            snap, _ = SOFT.all_nodes_case()
        finally:
            SOFT.NODEORDER_ARGS["tainttoleration.weight"] = 3
        snap.preempt_args = PreemptArguments(topology_aware=True, min_candidate_nodes_percentage=100,
                                             min_candidate_nodes_absolute=4, max_candidate_nodes_absolute=100)
        snap.preempt_seed, snap.now_ns = 0, 0
        for restated in (True, False):
            out.append(SC.statements(snap, S.run(snap, restated=restated).preempt))
    assert all(o == out[0] for o in out) and out[0]
