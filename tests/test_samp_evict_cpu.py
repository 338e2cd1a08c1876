"""Preempt and reclaim under feasible-node sampling on the CPU: the sampling oracle (tools/samp_evict_oracle) against the
unchanged oracle and topology oracle where sampling is off, the library's per-task NodesFitErrors kind (compiled by g++)
against the oracle's record, and a hand-derived chain of PredicateNodes calls."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import samp_cases as SC
from tests import samp_common as S

HERE = os.path.dirname(os.path.abspath(__file__))
SHIM_SRC = os.path.join(HERE, "hostshim", "samp_shim.cpp")
SHIM_OUT = os.path.join(HERE, "hostshim", "_build", "samp_shim.so")


@pytest.mark.parametrize("family", ["normal", "topo"])
def test_restated_actions_match_the_oracle_without_sampling(family):
    """At percentage-nodes-to-find 100 the restated actions (their own loops, PredicateNodes in NodeList order) give the
    statements and visits of oracle.cpp's preempt / reclaim and of the topology oracle's preempt."""
    from tools.fuzz_evict import make_case, make_topo_case
    checked = 0
    for seed in range(120):
        if family == "topo":
            tc, tiers, actions, conf = make_topo_case(seed)
        else:
            (tc, tiers, actions), conf = make_case(seed), {}
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        assert S.same(S.run(snap), S.run(snap, restated=False), index=False), seed
        checked += 1
    assert checked > 80


@pytest.fixture(scope="module")
def shim():
    os.makedirs(os.path.dirname(SHIM_OUT), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", SHIM_SRC, "-o", SHIM_OUT], check=True)
    L = C.CDLL(SHIM_OUT)
    L.vss_fit_error_node_kinds.argtypes = [C.POINTER(C.c_int32), C.c_size_t, C.POINTER(C.c_int32), C.POINTER(C.c_uint32),
                                           C.c_size_t, C.POINTER(C.c_uint8)]
    return L


def test_fit_error_kinds_match_the_oracle(shim):
    """Random allocate runs with named and unnamed roles (several pending tasks per role, selectors no node satisfies):
    the library's derivation from the fit-error list equals the kind the oracle records, and both kinds occur."""
    from tools.fuzz_evict import make_samp_case
    seen = set()
    for seed in range(200):
        tc, tiers, actions, conf = make_samp_case(seed)
        for k, p in enumerate(tc.Pods):
            if not p.node_name and k % 3 == 0:
                p.node_selector = {"zone": "nowhere"}
        snap = tc.RegisterSession(tiers, actions=("allocate", "preempt"), **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        o = S.SampOracle(snap)
        try:
            fe = o.allocate().fit_errors.astype(np.int32)
            want = o.node_errors()
        finally:
            o.close()
        got = np.zeros(max(snap.T, 1), np.uint8)
        t_role = np.ascontiguousarray(snap.t_role, np.int32)
        r_flags = np.ascontiguousarray(snap.r_flags, np.uint32)
        shim.vss_fit_error_node_kinds(fe.ctypes.data_as(C.POINTER(C.c_int32)), len(fe), t_role.ctypes.data_as(C.POINTER(C.c_int32)),
                                      r_flags.ctypes.data_as(C.POINTER(C.c_uint32)), snap.T, got.ctypes.data_as(C.POINTER(C.c_uint8)))
        assert np.array_equal(got[:snap.T], want), seed
        for t in fe:
            seen.add(int(want[t]))
    assert seen == {0, 1}


def test_hand_derived_predicate_nodes_chain():
    """Five 1-CPU nodes, n1 and n3 labelled zone=a, the others zone=b; one starving job (minMember 1, Inqueue) of five
    2-CPU pending pods, so nothing fits anywhere; percentage 50, min-nodes-to-find 1 (numNodesToFind(5) = 2 < 5: sampling
    is on); lastProcessedNodeIndex 7 (>= N); actions allocate, reclaim; no running pod, so every reclaimer fails.
    Task order (priority): e (40, role w, PreemptionPolicy Never), c (30, role x, zone=a), b (20, role x, zone=a),
    a (10, role y), d (5, role z, zone=c, a zone no node has).

    allocate (allocate.go:599-647): NeedContinueAllocating holds (minMember 1 < 5 tasks, no role minimum), so every task
    is visited. e, c, a and d fail the predicate on every node: entries with node errors. b's role x already has an entry:
    TaskHasFitErrors skips it, an entry without node errors, so b keeps the whole NodeList. Each failing scan visits all 5
    nodes from 7: the index becomes (7 + 5) % 5 = 2.
    reclaim (reclaim.go:140-180, predicate_helper.go:43-140), from 2:
      e: PreemptionPolicy Never returns before PredicateNodes: no call, the index stays 2.
      c: filtered list = static-feasible nodes [n1, n3], P = 2, numNodesToFind(2) = 1; start 2 >= P visits list[2 % 2] = n1,
         which passes: predicateNodes [n1], processed 1, index (2 + 1) % 2 = 1.
      b: whole NodeList, P = 5, numNodesToFind 2; from 1: n1 passes, n2 fails (zone b), n3 passes: [n1, n3],
         processed 3, index (1 + 3) % 5 = 4.
      a: filtered list = every node (no selector), P = 5; from 4: n4, n0 pass (wrap-around): [n4, n0], processed 2,
         index (4 + 2) % 5 = 1.
      d: filtered list empty: returns early, the index stays 1."""
    from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList
    from volcano_b200.snapshot import PluginOption
    from volcano_b200.uthelper import TestCommonStruct
    nodes = [BuildNode(f"n{i}", BuildResourceList("1", "1G", ("pods", "10")), {"zone": "a" if i in (1, 3) else "b"})
             for i in range(5)]
    spec = [("e", 40, "w", None), ("c", 30, "x", "a"), ("b", 20, "x", "a"), ("a", 10, "y", None), ("d", 5, "z", "c")]
    pods = []
    for name, prio, role, zone in spec:
        p = BuildPod("ns", name, "", "Pending", BuildResourceList("2", "1G"), "pg", {"volcano.sh/task-spec": role},
                     {"zone": zone} if zone else {})
        p.priority = prio
        if name == "e":
            p.preemption_policy = "Never"
        pods.append(p)
    tc = TestCommonStruct(Name="samp-chain", Nodes=nodes, Pods=pods, PodGroups=[BuildPodGroup("pg", "ns", "q", 1, None, "Inqueue")],
                          Queues=[BuildQueue("q", 1, None)])
    tiers = [[PluginOption.defaults("priority"), PluginOption.defaults("gang"), PluginOption.defaults("predicates")]]
    snap = tc.RegisterSession(tiers, actions=("allocate", "reclaim"), percentage_nodes_to_find=50, min_nodes_to_find=1,
                              last_processed_node_index=7, enable_predicate_error_cache=False)
    t = {k.split("/")[-1]: i for i, k in enumerate(snap.task_keys)}
    kept = {}
    res = S.run(snap, keep=lambda o: kept.update(calls=o.calls(), kinds=o.node_errors()))
    assert [int(kept["kinds"][t[n]]) for n in "ecbad"] == [1, 1, 0, 1, 1]
    assert kept["calls"] == [
        {"task": t["c"], "P": 2, "processed": 1, "index": 1, "nodes": [1]},
        {"task": t["b"], "P": 5, "processed": 3, "index": 4, "nodes": [1, 3]},
        {"task": t["a"], "P": 5, "processed": 2, "index": 1, "nodes": [4, 0]},
        {"task": t["d"], "P": 0, "processed": 0, "index": 1, "nodes": []},
    ]
    assert res.reclaim.stats["last_processed_node_index"] == 1
    assert len(res.reclaim.decisions) == 0


@pytest.mark.parametrize("case", sorted(SC.CASES))
def test_hand_derived_cases(case):
    """tests/samp_cases.py, each derived from the Go code in its builder's docstring: the PredicateNodes calls of preempt
    and reclaim (task, P, processed, index after, predicateNodes in scan order), the index each action leaves and its
    statements. chain: the index through allocate, preempt's inter- and intra-job phases and reclaim, a full scan that
    rewrites the index modulo P, taskEligibleToPreempt and reclaim's Never check leaving it alone; tie: SortNodes' equal
    scores in scan order; reclaim: a reclaim on the first node in scan order; topo: the offset counted in scan order."""
    snap, exp = SC.CASES[case]()
    kept = {}
    res = S.run(snap, keep=lambda o: kept.update(calls=o.calls()))
    assert kept["calls"] == SC.expected_calls(snap, exp["calls"])
    for action, idx in exp["index"].items():
        r = getattr(res, action)
        assert r.stats["last_processed_node_index"] == idx, action
        assert SC.statements(snap, r) == exp[action], action


def test_hand_derived_entry_kinds(shim):
    """tests/samp_cases.kinds_case: two named roles with a failing and a skipped task each, and three failing tasks of the
    empty role. The oracle's record and the library's derivation from the fit-error list both give the derived kinds."""
    snap, exp = SC.kinds_case()
    o = S.SampOracle(snap)
    try:
        fe = o.allocate().fit_errors.astype(np.int32)
        kinds = o.node_errors()
    finally:
        o.close()
    assert {n: int(kinds[SC.task_index(snap, n)]) for n in exp} == exp
    got = np.zeros(snap.T, np.uint8)
    t_role = np.ascontiguousarray(snap.t_role, np.int32)
    r_flags = np.ascontiguousarray(snap.r_flags, np.uint32)
    shim.vss_fit_error_node_kinds(fe.ctypes.data_as(C.POINTER(C.c_int32)), len(fe), t_role.ctypes.data_as(C.POINTER(C.c_int32)),
                                  r_flags.ctypes.data_as(C.POINTER(C.c_uint32)), snap.T, got.ctypes.data_as(C.POINTER(C.c_uint8)))
    assert {n: int(got[SC.task_index(snap, n)]) for n in exp} == exp
