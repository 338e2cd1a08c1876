"""Preempt and reclaim under feasible-node sampling on the H100: k_evict_samp launched on its own against a numpy
restatement of PredicateNodes, and whole sessions (allocate -> preempt -> reclaim, both readings of preempt) against the
sampling oracle (tools/samp_evict_oracle), statements, visits and the carried lastProcessedNodeIndex compared."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import samp_cases as SC
from tests import samp_common as S

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "tools", "kernels", "_build", "evict_harness.so")


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build() compiles it")
    L = C.CDLL(LIB)
    i32p = C.POINTER(C.c_int32)
    L.eh_samp.argtypes = [C.c_int, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int32, i32p, i32p, i32p]
    return L


def num_to_find(P, pct, min_nodes, min_pct):  # CalculateNumOfFeasibleNodesToFind, util/scheduler_helper.go:54-73
    if P <= min_nodes or pct >= 100:
        return P
    a = pct
    if a <= 0:
        a = max(50 - P // 125, min_pct)
    return max(P * a // 100, min_nodes)


def restated(passes, filtered, pct, min_nodes, min_pct, start):
    """PredicateNodes over the (filtered) NodeList, single-worker reading: (nodes in scan order, index after)."""
    nodes = np.flatnonzero(passes) if filtered else np.arange(len(passes))
    P = len(nodes)
    if P == 0:
        return [], start
    tf = num_to_find(P, pct, min_nodes, min_pct)
    order = nodes[(start + np.arange(P)) % P]
    ok = passes[order].astype(bool)
    found = np.flatnonzero(ok)
    processed = P if len(found) < tf else int(found[tf - 1]) + 1
    return [int(n) for n in order[found[:tf]]], (start + processed) % P


CASES = []
for _N in (1, 2, 101, 1000, 10_001, 200_000):
    for _kind in ("random", "fail", "pass", "sparse"):
        CASES.append((_N, _kind))


@pytest.mark.parametrize("N,kind", CASES)
def test_samp_kernel_matches_restatement(H, N, kind):
    """Random verdicts, all-fail, all-pass and 1 % passing; both list readings; `start` below N, at N and beyond (up to
    3N); numNodesToFind = 1, numNodesToFind = P with fewer passing nodes (min-nodes-to-find above N), and the adaptive
    percentage."""
    rng = np.random.default_rng(N * 7 + len(kind))
    p = {"random": 0.5, "fail": 0.0, "pass": 1.0, "sparse": 0.01}[kind]
    passes = (rng.random(N) < p).astype(np.uint8)
    args = [(0, 1, 5), (1, 1, 5), (100, 1, 5), (0, 100, 5), (50, 1, 5), (5, 10 ** 6, 5), (0, 1, 100)]
    for pct, min_nodes, min_pct in args:
        for filtered in (0, 1):
            for start in sorted({0, 1, N - 1, N, N + 3, 3 * N, int(rng.integers(0, 3 * N + 1))}):
                if start < 0:
                    continue
                lst = np.full(N, -7, np.int32)
                cnt, idx = C.c_int32(0), C.c_int32(0)
                i32p = C.POINTER(C.c_int32)
                assert H.eh_samp(N, passes.ctypes.data_as(C.POINTER(C.c_uint8)), filtered, pct, min_nodes, min_pct, start,
                                 lst.ctypes.data_as(i32p), C.byref(cnt), C.byref(idx)) == 0
                want, want_idx = restated(passes, filtered, pct, min_nodes, min_pct, start)
                got = [int(x) for x in lst[:cnt.value]]
                assert got == want, (N, kind, pct, min_nodes, filtered, start)
                assert idx.value == want_idx, (N, kind, pct, min_nodes, filtered, start, idx.value, want_idx)


def _gpu(snap):
    from volcano_b200 import engine
    engine.init(0)
    return engine.gpu_engine(snap)


def test_sessions_match_the_oracle():
    """320 random sessions of the sampling fuzz family (tools/fuzz_evict.make_samp_case), normal and topology-aware
    preempt: allocate placements, preempt / reclaim statements and visits, and the index after each evicting action
    identical."""
    from tools.fuzz_evict import make_samp_case
    checked = evictions = 0
    for seed in range(320):
        tc, tiers, actions, conf = make_samp_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = S.run(snap)
        res = _gpu(snap)
        assert S.same(res, ref), (seed, actions, conf)
        checked += 1
        evictions += sum(len(getattr(ref, a).decisions) for a in ("preempt", "reclaim") if getattr(ref, a) is not None)
    assert checked >= 250 and evictions > 0


@pytest.mark.parametrize("case", sorted(SC.CASES))
def test_hand_derived_cases(case):
    """The library on the hand-derived sessions of tests/samp_cases.py: the statements and the index each evicting action
    leaves are the values derived there from the Go code."""
    snap, exp = SC.CASES[case]()
    res = _gpu(snap)
    for action, idx in exp["index"].items():
        r = getattr(res, action)
        assert r.stats["last_processed_node_index"] == idx, action
        assert SC.statements(snap, r) == exp[action], action


def test_sampling_off_is_unchanged():
    """The same family at percentage-nodes-to-find 100: the library matches the unchanged oracle and the topology oracle
    (NodeList order, index untouched)."""
    from tools.fuzz_evict import make_samp_case
    for seed in range(60):
        tc, tiers, actions, conf = make_samp_case(seed)
        conf["percentage_nodes_to_find"] = 100
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        assert S.same(_gpu(snap), S.run(snap, restated=False), index=False), seed


def test_impure_roles_with_error_cache_are_refused():
    """Sampling + enablePredicateErrorCache + a job whose named role spans two (class, request) groups: VC_EUNSUPPORTED
    from preempt, where the whole sampling mode was refused before."""
    from volcano_b200 import engine
    from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList
    from volcano_b200.snapshot import PluginOption
    from volcano_b200.uthelper import TestCommonStruct
    nodes = [BuildNode(f"n{i}", BuildResourceList("1", "1G", ("pods", "10"))) for i in range(4)]
    pods = [BuildPod("ns", f"p{k}", "", "Pending", BuildResourceList(str(k + 1), "1G"), "pg",
                     {"volcano.sh/task-spec": "w"}) for k in range(2)]
    tc = TestCommonStruct(Name="impure", Nodes=nodes, Pods=pods, PodGroups=[BuildPodGroup("pg", "ns", "q", 1, None, "Inqueue")],
                          Queues=[BuildQueue("q", 1, None)])
    tiers = [[PluginOption.defaults("gang"), PluginOption.defaults("priority"), PluginOption.defaults("predicates")]]
    snap = tc.RegisterSession(tiers, actions=("allocate", "preempt"), percentage_nodes_to_find=50, min_nodes_to_find=1,
                              enable_predicate_error_cache=True)
    engine.init(0)
    e = engine.Engine(snap)
    try:
        e.upload()
        e.allocate()
        with pytest.raises(Exception, match="enablePredicateErrorCache|-2|UNSUPPORTED"):
            e.preempt()
    finally:
        e.close()


def test_full_size_cfg5_adaptive_sampling():
    """A full-size cfg5 session (10 000 nodes) under the reference's default adaptive sampling (5 % at 10 000 nodes):
    allocate -> preempt -> reclaim, normal and topology-aware readings, statements and index identical to the oracle."""
    from volcano_b200.snapshot import PreemptArguments
    from volcano_b200.synth import make_cfg5
    for topo in (False, True):
        snap = make_cfg5(seed=1000)
        snap.conf.percentage_nodes_to_find = 0
        snap.conf.min_nodes_to_find = 100
        snap.conf.min_percentage_nodes_to_find = 5
        snap.conf.enable_predicate_error_cache = 0
        if topo:
            snap.preempt_args = PreemptArguments(topology_aware=True)
            snap.preempt_seed, snap.now_ns = 12345, 10 ** 9
        ref = S.run(snap)
        res = _gpu(snap)
        assert S.same(res, ref), topo
        assert ref.preempt is not None and ref.reclaim is not None
