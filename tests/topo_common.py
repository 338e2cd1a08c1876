"""Topology-aware preemption (the preempt action's enableTopologyAwarePreemption) test support: the oracle extension's
loader, an engine callable over it, and hand-derived sessions. The upstream cases are in tests/golden/topo_preempt_cases.py."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from volcano_b200 import abi
from tests.golden.topo_preempt_cases import PREEMPTABLE, _node
from volcano_b200.api import BuildPod, BuildPodGroupWithPrio, BuildQueue, BuildResourceList
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import AllocateResult, TestCommonStruct

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = os.path.join(ROOT, "tools", "topo_oracle", "_build", "libtopo_oracle.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        import __graft_entry__
        from oracle import pyoracle
        __graft_entry__.build_topo_oracle()
        L = C.CDLL(_LIB)  # oracle.cpp's C interface + the vcot_* functions
        ref = pyoracle.lib()
        for name in ("vco_session_create", "vco_session_destroy", "vco_session_set_running", "vco_allocate_run",
                     "vco_reclaim", "vco_num_decisions", "vco_num_visits", "vco_num_fit_errors", "vco_decisions",
                     "vco_visits", "vco_fit_errors"):
            getattr(L, name).restype = getattr(ref, name).restype
            getattr(L, name).argtypes = getattr(ref, name).argtypes
        L.vcot_set_preempt_options.argtypes = [C.c_void_p, C.POINTER(abi.vc_preempt_options)]
        L.vcot_preempt.argtypes = [C.c_void_p]
        L.vcot_forget.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class TopoOracle:
    """A CPU oracle session whose preempt action reads the snapshot's preempt options."""

    def __init__(self, snap):
        L = lib()
        self.snap = snap
        d, n, t, c, j, q = snap.dims(), snap.nodes(), snap.tasks(), snap.classes(), snap.jobs(), snap.queues()
        self.h = L.vco_session_create(C.byref(d), C.byref(n), C.byref(t), C.byref(c), C.byref(j), C.byref(q),
                                      C.byref(snap.conf), 1)
        assert self.h
        rt = snap.running_tasks()
        if rt is not None or snap.t_flags.any():
            tf = snap.t_flags.ctypes.data_as(C.POINTER(C.c_uint32)) if snap.T else None
            assert L.vco_session_set_running(self.h, C.byref(rt) if rt is not None else None, tf) == 0
        po = snap.preempt_options()
        assert L.vcot_set_preempt_options(self.h, C.byref(po) if po is not None else None) == 0

    def close(self):
        if self.h:
            lib().vcot_forget(self.h)
            lib().vco_session_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _run(self, fn, what):
        rc = fn(self.h)
        if rc != 0:
            raise RuntimeError(f"topo oracle {what} rc={rc}")
        from oracle.pyoracle import DECISION_DTYPE, VISIT_DTYPE
        L = lib()
        nd, nv = L.vco_num_decisions(self.h), L.vco_num_visits(self.h)
        dec = np.ctypeslib.as_array(C.cast(L.vco_decisions(self.h), C.POINTER(C.c_uint8)), (nd * DECISION_DTYPE.itemsize,)
                                    ).view(DECISION_DTYPE).copy() if nd else np.zeros(0, DECISION_DTYPE)
        vis = np.ctypeslib.as_array(C.cast(L.vco_visits(self.h), C.POINTER(C.c_uint8)), (nv * VISIT_DTYPE.itemsize,)
                                    ).view(VISIT_DTYPE).copy() if nv else np.zeros(0, VISIT_DTYPE)
        return AllocateResult(dec, vis, np.zeros(0, np.int32))

    def allocate(self):
        return self._run(lib().vco_allocate_run, "allocate")

    def preempt(self):
        return self._run(lib().vcot_preempt, "preempt")

    def reclaim(self):
        return self._run(lib().vco_reclaim, "reclaim")


def oracle_engine(snap) -> AllocateResult:
    """Snapshot -> AllocateResult through the topology-aware oracle, the configured actions in order."""
    o = TopoOracle(snap)
    try:
        actions = [a for a in snap.actions if a != "enqueue"]
        if "allocate" in actions:
            res = o.allocate()
        else:
            res = AllocateResult(np.zeros(0, abi_decision()), np.zeros(0, abi_visit()), np.zeros(0, np.int32))
        for a in actions:
            if a == "preempt":
                res.preempt = o.preempt()
            elif a == "reclaim":
                res.reclaim = o.reclaim()
        return res
    finally:
        o.close()


def abi_decision():
    from oracle.pyoracle import DECISION_DTYPE
    return DECISION_DTYPE


def abi_visit():
    from oracle.pyoracle import VISIT_DTYPE
    return VISIT_DTYPE


def same(a: AllocateResult, b: AllocateResult) -> bool:
    """Identical decisions and visits of every action."""
    for name in ("preempt", "reclaim"):
        x, y = getattr(a, name), getattr(b, name)
        if (x is None) != (y is None):
            return False
        if x is not None and not (np.array_equal(x.decisions, y.decisions) and np.array_equal(x.visits, y.visits)):
            return False
    return np.array_equal(a.decisions["task"], b.decisions["task"]) and np.array_equal(a.decisions["node"], b.decisions["node"])


def _tiers(proportion_predicate=True):
    return [[PluginOption.make("priority", EnabledTaskOrder=True, EnabledJobOrder=True, EnabledPreemptable=True,
                               EnabledJobStarving=True),
             PluginOption.make("gang", EnabledJobPipelined=True, EnabledJobStarving=True),
             PluginOption.make("proportion", EnabledAllocatable=True, EnabledQueueOrder=True,
                               EnabledPredicate=proportion_predicate)]]


def _pod(name, node, cpu, pg, prio=None, start=None, task_prio=None):
    p = BuildPod("c1", name, node, "Running" if node else "Pending", BuildResourceList(cpu, f"{cpu}G"), pg, PREEMPTABLE)
    p.priority = prio
    p.start_time = start
    if task_prio is not None:
        p.annotations["volcano.sh/task-priority"] = str(task_prio)
    return p


def hand_cases():
    """Hand-derived sessions, one per rule of the topology-aware reading: (TestCommonStruct, tiers, RegisterSession
    keyword arguments). Each case's docstring-like Name states the derivation; ExpectEvicted / ExpectPipeLined hold it."""
    def topo(pct=100, min_abs=1, max_abs=100, seed=0, now=0):
        return {"configurations": {"preempt": {"enableTopologyAwarePreemption": True, "minCandidateNodesPercentage": pct,
                                               "minCandidateNodesAbsolute": min_abs, "maxCandidateNodesAbsolute": max_abs}},
                "preempt_seed": seed, "now_ns": now}
    pgs = lambda *extra: [BuildPodGroupWithPrio("pg1", "c1", "q1", 1, None, "Running", 10),
                          BuildPodGroupWithPrio("pg2", "c1", "q1", 1, None, "Inqueue", 1000), *extra]
    cases = []
    # 1. the preemptor already fits: its one victim is popped (nothing is tested before the first removal), then
    #    reprieved, so the node has no victim and is no candidate: nothing is evicted and nothing pipelined (the normal
    #    reading pipelines the preemptor there without evictions)
    cases.append((TestCommonStruct(
        Name="already fits: popped, reprieved, no candidate", PodGroups=pgs(), Queues=[BuildQueue("q1", 1, None)],
        Nodes=[_node("n1", "10", "10G")], Pods=[_pod("v1", "n1", "1", "pg1"), _pod("pre", "", "1", "pg2")],
        ExpectEvicted=[], ExpectEvictNum=0, ExpectPipeLined={}), _tiers(), topo()))
    # 2. the queue's quota fails even with both victims gone (cap 3, preemptor 4): every popped task stays a victim and
    #    the preemptor is pipelined over quota (ValidateVictims checks resources only)
    cases.append((TestCommonStruct(
        Name="quota exceeded: every popped task stays a victim, preemptor pipelined", PodGroups=pgs(),
        Queues=[BuildQueue("q1", 1, BuildResourceList("3", "3G"))], Nodes=[_node("n1", "4", "4G")],
        Pods=[_pod("v1", "n1", "1", "pg1"), _pod("v2", "n1", "1", "pg1"), _pod("pre", "", "4", "pg2")],
        ExpectEvicted=["c1/v1", "c1/v2"], ExpectEvictNum=2, ExpectPipeLined={"c1/pg2": ["n1"]}), _tiers(), topo()))
    # 3. proportion without EnabledPredicate: its PrePredicateFn never writes the state, SimulateRemoveTaskFn fails on
    #    every node, so no node is a candidate
    cases.append((TestCommonStruct(
        Name="proportion without EnabledPredicate: no candidate", PodGroups=pgs(), Queues=[BuildQueue("q1", 1, None)],
        Nodes=[_node("n1", "2", "2G")], Pods=[_pod("v1", "n1", "2", "pg1"), _pod("pre", "", "2", "pg2")],
        ExpectEvicted=[], ExpectEvictNum=0, ExpectPipeLined={}), _tiers(False), topo()))
    # 4. numCandidates = 4 * 50 / 100 = 2 of 4 nodes with one victim each (pod priorities 50, 1, 1, 40). Seed 0 gives
    #    offset splitmix64(0) % 4 = 3: the candidates are n3, then n0 (wrap-around), and the lower highest victim
    #    priority wins: n3. Seed 6 gives offset 0: candidates n0, n1, winner n1.
    four = [_node(f"n{i}", "2", "2G") for i in range(4)]
    four_pods = [_pod(f"v{i}", f"n{i}", "2", "pg1", prio=p) for i, p in enumerate((50, 1, 1, 40))]
    for seed, node in ((0, "n3"), (6, "n1")):
        cases.append((TestCommonStruct(
            Name=f"numCandidates cut, seed {seed}: winner {node}", PodGroups=pgs(), Queues=[BuildQueue("q1", 1, None)],
            Nodes=four, Pods=four_pods + [_pod("pre", "", "2", "pg2")],
            ExpectEvicted=[f"c1/v{node[1]}"], ExpectEvictNum=1, ExpectPipeLined={"c1/pg2": [node]}),
            _tiers(), topo(pct=50, seed=seed)))
    # 5. victims[0] is the list's first element, not the highest-priority victim: on n0 the victims of job pg3 (job
    #    priority 5, pod priority 100) pop before pg1's (job priority 10, pod priority 1); both are needed, and the
    #    reprieve walks back, so the list is [v01 (1), v00 (100)] and n0 scores -1 against n1's -50: n0 wins
    two = [_node("n0", "2", "2G"), _node("n1", "2", "2G")]
    cases.append((TestCommonStruct(
        Name="victims[0] literally: the last popped victim", Queues=[BuildQueue("q1", 1, None)], Nodes=two,
        PodGroups=pgs(BuildPodGroupWithPrio("pg3", "c1", "q1", 1, None, "Running", 5)),
        Pods=[_pod("v00", "n0", "1", "pg3", prio=100), _pod("v01", "n0", "1", "pg1", prio=1),
              _pod("v10", "n1", "2", "pg1", prio=50), _pod("pre", "", "2", "pg2")],
        ExpectEvicted=["c1/v00", "c1/v01"], ExpectEvictNum=2, ExpectPipeLined={"c1/pg2": ["n0"]}), _tiers(), topo()))
    # 6. the sum key with its 2^31 term: n0's victims [5, -10] sum to -5 + 2 * 2^31, n1's [5] to 5 + 2^31; the first
    #    keys tie (-5), the smaller sum wins: n1 (without the 2^31 term n0 would)
    cases.append((TestCommonStruct(
        Name="sum of priorities with the 2^31 term decides", Queues=[BuildQueue("q1", 1, None)], Nodes=two, PodGroups=pgs(),
        Pods=[_pod("v00", "n0", "1", "pg1", prio=5), _pod("v01", "n0", "1", "pg1", prio=-10),
              _pod("v10", "n1", "2", "pg1", prio=5), _pod("pre", "", "2", "pg2")],
        ExpectEvicted=["c1/v10"], ExpectEvictNum=1, ExpectPipeLined={"c1/pg2": ["n1"]}), _tiers(), topo()))
    # 7. the start-time key: equal priorities and counts; n0's victim started at 2 s, n1's has no StartTime and takes
    #    now_ns. now = 3 s: n1 started latest and wins; now = 1 s: n0 wins
    for now, node in ((3 * 10 ** 9, "n1"), (10 ** 9, "n0")):
        cases.append((TestCommonStruct(
            Name=f"latest start time, nil start at now={now}: winner {node}", Queues=[BuildQueue("q1", 1, None)],
            Nodes=two, PodGroups=pgs(),
            Pods=[_pod("v0", "n0", "2", "pg1", prio=5, start=2 * 10 ** 9), _pod("v1", "n1", "2", "pg1", prio=5),
                  _pod("pre", "", "2", "pg2")],
            ExpectEvicted=[f"c1/v{node[1]}"], ExpectEvictNum=1, ExpectPipeLined={"c1/pg2": [node]}), _tiers(), topo(now=now)))
    # 8. ties on every score fall to the candidate order: seed 0 gives offset splitmix64(0) % 2 = 1, so n1 is the first
    #    candidate and wins over the identical n0
    cases.append((TestCommonStruct(
        Name="full tie: the first candidate in scan order wins", Queues=[BuildQueue("q1", 1, None)], Nodes=two, PodGroups=pgs(),
        Pods=[_pod("v0", "n0", "2", "pg1", prio=5, start=10 ** 9), _pod("v1", "n1", "2", "pg1", prio=5, start=10 ** 9),
              _pod("pre", "", "2", "pg2")],
        ExpectEvicted=["c1/v1"], ExpectEvictNum=1, ExpectPipeLined={"c1/pg2": ["n1"]}), _tiers(), topo(seed=0)))
    # 9. PodPriority, not TaskInfo.Priority: n0's victim has pod priority 5 and task priority 100 (annotation), n1's pod
    #    priority 10: n0 wins on -5 > -10
    cases.append((TestCommonStruct(
        Name="PodPriority, not TaskInfo.Priority", Queues=[BuildQueue("q1", 1, None)], Nodes=two, PodGroups=pgs(),
        Pods=[_pod("v0", "n0", "2", "pg1", prio=5, task_prio=100), _pod("v1", "n1", "2", "pg1", prio=10),
              _pod("pre", "", "2", "pg2")],
        ExpectEvicted=["c1/v0"], ExpectEvictNum=1, ExpectPipeLined={"c1/pg2": ["n0"]}), _tiers(), topo()))
    return cases
