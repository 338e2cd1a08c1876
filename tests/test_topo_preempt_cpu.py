"""Topology-aware preemption on the CPU: the upstream TestTopologyAwarePreempt cases and hand-derived sessions on the
oracle's restatement (tools/topo_oracle), and the preempt action's argument parsing."""
import pytest

from tests import topo_common as X
from tests.golden import topo_preempt_cases as G
from volcano_b200 import abi
from volcano_b200.snapshot import PreemptArguments, SchedulerConf, preempt_arguments


@pytest.mark.parametrize("case", G.golden_cases(), ids=lambda c: c.Name[:50])
def test_topology_aware_goldens(case):
    """actions/preempt/preempt_test.go:427-747 (9 of 12 cases) with enableTopologyAwarePreemption: true."""
    case.RegisterSession(G.topo_tiers(), actions=("preempt",), configurations=G.TOPO, preempt_seed=1, now_ns=0)
    case.Run(X.oracle_engine)
    assert case.CheckAll() is None, case.CheckAll()


@pytest.mark.parametrize("case,tiers,kw", X.hand_cases(), ids=lambda c: getattr(c, "Name", "")[:50])
def test_hand_derived(case, tiers, kw):
    case.RegisterSession(tiers, actions=("preempt",), **kw)
    case.Run(X.oracle_engine)
    assert case.CheckAll() is None, case.CheckAll()


def test_normal_reading_differs_on_the_hand_cases():
    """The first two hand cases come out differently in the normal reading: the preemptor that already fits is
    pipelined without evictions, and the over-quota one is discarded."""
    got = []
    for case, tiers, kw in X.hand_cases()[:2]:
        kw = dict(kw, configurations={})
        case.RegisterSession(tiers, actions=("preempt",), **kw)
        case.Run(X.oracle_engine)
        got.append((sorted(case.evicts), case.pipelined))
    assert got == [([], {"c1/pg2": ["n1"]}), ([], {})]


def test_arguments_read_like_framework_arguments():
    """GetBool / GetInt type-assert: a bool and ints are taken, strings (even "true" / "30") and bools for ints keep
    the defaults."""
    conf = SchedulerConf(tiers=[], configurations={"preempt": {
        "enableTopologyAwarePreemption": True, "minCandidateNodesPercentage": 30, "minCandidateNodesAbsolute": "2",
        "maxCandidateNodesAbsolute": True, "topologyAwarePreemptWorkerNum": 4}})
    a = preempt_arguments(conf)
    assert (a.topology_aware, a.min_candidate_nodes_percentage, a.min_candidate_nodes_absolute,
            a.max_candidate_nodes_absolute, a.worker_num) == (True, 30, 1, 100, 4)
    assert not preempt_arguments(SchedulerConf(tiers=[], configurations={"preempt": {
        "enableTopologyAwarePreemption": "true"}})).topology_aware
    assert preempt_arguments(SchedulerConf(tiers=[])) == PreemptArguments()


def test_negative_candidate_count_is_refused():
    """maxCandidateNodesAbsolute < 0 makes numCandidates negative: the reference panics in make."""
    case = G.golden_cases()[2]
    case.RegisterSession(G.topo_tiers(), actions=("preempt",),
                         configurations={"preempt": {"enableTopologyAwarePreemption": True, "maxCandidateNodesAbsolute": -1}})
    with pytest.raises(RuntimeError, match=f"rc={abi.VC_EINVAL}$"):
        case.Run(X.oracle_engine)
