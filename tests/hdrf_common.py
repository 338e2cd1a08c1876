"""Hierarchical drf (drf's enableHierarchy) test support: the oracle extension's loader and the sessions the hdrf tests use.

The upstream cases are transcribed from plugins/drf/hdrf_test.go (TestHDRF). Its assertion,
`if equality.Semantic.DeepEqual(test.expected, job.Allocated) { t.Fatalf(...) }`, compares the whole expected map with ONE
job's *Resource: the two never compare equal, so the test can never fail. The expected tables are the authors' intent and
were never checked; the tests here state what the reference's code actually computes.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueueWithAnnos, BuildResourceList
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = os.path.join(ROOT, "tools", "hdrf_oracle", "_build", "libhdrf_oracle.so")
_lib = None
_dp, _i32p = C.POINTER(C.c_double), C.POINTER(C.c_int32)
HIER, WEIGHTS = "volcano.sh/hierarchy", "volcano.sh/hierarchy-weights"


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        import __graft_entry__
        from volcano_b200 import abi
        __graft_entry__.build_hdrf_oracle()
        L = C.CDLL(_LIB)  # oracle.cpp's C interface + the vcoh_* functions
        L.vco_session_create.restype = C.c_void_p
        L.vco_session_create.argtypes = [C.POINTER(abi.vc_dims), C.POINTER(abi.vc_nodes), C.POINTER(abi.vc_tasks),
                                         C.POINTER(abi.vc_classes), C.POINTER(abi.vc_jobs), C.POINTER(abi.vc_queues),
                                         C.POINTER(abi.vc_conf), C.c_int]
        L.vco_session_destroy.argtypes = [C.c_void_p]
        L.vcoh_attach.argtypes = [C.c_void_p, C.c_char_p, _i32p, _dp, _dp]
        L.vcoh_detach.argtypes = [C.c_void_p]
        L.vcoh_allocate_run.argtypes = [C.c_void_p, C.c_int]
        L.vcoh_backfill.argtypes = [C.c_void_p]
        L.vcoh_backfill_pick_order.argtypes = [C.c_void_p, _i32p]
        L.vco_session_set_backfill.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.vc_tasks)]
        L.vcoh_compare.restype = C.c_double
        L.vcoh_compare.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.vcoh_node.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp, _dp, C.POINTER(C.c_int), _dp]
        L.vcoh_job_add.argtypes = [C.c_void_p, C.c_int, _dp]
        for n in ("vco_num_decisions", "vco_num_visits", "vco_num_fit_errors"):
            getattr(L, n).restype = C.c_size_t
            getattr(L, n).argtypes = [C.c_void_p]
        L.vco_decisions.restype = C.c_void_p
        L.vco_visits.restype = C.c_void_p
        L.vco_fit_errors.restype = _i32p
        for n in ("vco_decisions", "vco_visits", "vco_fit_errors"):
            getattr(L, n).argtypes = [C.c_void_p]
        _lib = L
    return _lib


class HdrfOracle:
    """A CPU oracle session with drf's enableHierarchy: the hierarchy / weights annotation strings of every queue."""

    def __init__(self, snap, hierarchy, weights, threads: int = 1):
        from volcano_b200 import abi
        from volcano_b200.snapshot import go_parse_float
        L = lib()
        self.snap = snap
        d, n, t, c, j, q = snap.dims(), snap.nodes(), snap.tasks(), snap.classes(), snap.jobs(), snap.queues()
        self.h = L.vco_session_create(C.byref(d), C.byref(n), C.byref(t), C.byref(c), C.byref(j), C.byref(q),
                                      C.byref(snap.conf), threads)
        assert self.h
        # the same session set-up as oracle.pyoracle.OracleSession: topology, BestEffort list, nominated nodes, node.Tasks
        topo = snap.topology()
        if topo is not None:
            L.vco_session_set_topology.argtypes = [C.c_void_p, C.POINTER(abi.vc_hypernodes)]
            L.vco_session_set_topology(self.h, C.byref(topo))
        bt = snap.backfill_tasks()
        if bt is not None:
            assert L.vco_session_set_backfill(self.h, snap.B, C.byref(bt)) == 0
        nom = getattr(snap, "t_nominated", None)
        if nom is not None and snap.T and (nom >= 0).any():
            L.vco_session_set_nominated.argtypes = [C.c_void_p, _i32p]
            L.vco_session_set_nominated(self.h, np.ascontiguousarray(nom, np.int32).ctypes.data_as(_i32p))
        rt = snap.running_tasks()
        if rt is not None or snap.t_flags.any():
            L.vco_session_set_running.argtypes = [C.c_void_p, C.POINTER(abi.vc_running_tasks), C.POINTER(C.c_uint32)]
            tf = snap.t_flags.ctypes.data_as(C.POINTER(C.c_uint32)) if snap.T else None
            assert L.vco_session_set_running(self.h, C.byref(rt) if rt is not None else None, tf) == 0
        nw = np.array([len(w.split("/")) for w in weights], np.int32)
        wv = np.array([go_parse_float(x) for w in weights for x in w.split("/")] or [0.0], np.float64)
        jr = np.ascontiguousarray(snap.hd_job_request if snap.hdrf() is not None else np.zeros((snap.R, snap.J)))
        self.attach_rc = L.vcoh_attach(self.h, "\n".join(hierarchy).encode(), nw.ctypes.data_as(_i32p),
                                       wv.ctypes.data_as(_dp), jr.ctypes.data_as(_dp))

    def __del__(self):
        try:
            lib().vcoh_detach(self.h)
            lib().vco_session_destroy(self.h)
        except Exception:
            pass

    def allocate(self, argmin: bool = False):
        """allocate under hdrf; argmin=True replaces the queue heap by an arg-min over live keys (not the reference)."""
        rc = lib().vcoh_allocate_run(self.h, 1 if argmin else 0)
        if rc != 0:
            raise RuntimeError(f"hdrf oracle allocate rc={rc}")
        return self._results()

    def backfill(self):
        """backfill under hdrf on the state the session is in (after allocate())."""
        rc = lib().vcoh_backfill(self.h)
        if rc != 0:
            raise RuntimeError(f"hdrf oracle backfill rc={rc}")
        return self._results()

    def backfill_pick_order(self):
        out = np.zeros(max(self.snap.B, 1), np.int32)
        n = lib().vcoh_backfill_pick_order(self.h, out.ctypes.data_as(_i32p))
        return out[:n].copy()

    def _results(self):
        from oracle.pyoracle import DECISION_DTYPE, VISIT_DTYPE
        L = lib()
        nd, nv, nf = L.vco_num_decisions(self.h), L.vco_num_visits(self.h), L.vco_num_fit_errors(self.h)
        dec = np.ctypeslib.as_array(C.cast(L.vco_decisions(self.h), C.POINTER(C.c_uint8)), (nd * DECISION_DTYPE.itemsize,)
                                    ).view(DECISION_DTYPE).copy() if nd else np.zeros(0, DECISION_DTYPE)
        vis = np.ctypeslib.as_array(C.cast(L.vco_visits(self.h), C.POINTER(C.c_uint8)), (nv * VISIT_DTYPE.itemsize,)
                                    ).view(VISIT_DTYPE).copy() if nv else np.zeros(0, VISIT_DTYPE)
        fe = np.ctypeslib.as_array(L.vco_fit_errors(self.h), (nf,)).copy() if nf else np.zeros(0, np.int32)
        return dec, vis, fe

    def node(self, q: int, level: int):
        """(share, weight, saturated, allocated) of the node at `level` of queue q's path (0 = the root)."""
        s, w, sat = C.c_double(), C.c_double(), C.c_int()
        a = np.zeros(self.snap.R)
        assert lib().vcoh_node(self.h, q, level, C.byref(s), C.byref(w), C.byref(sat), a.ctypes.data_as(_dp)) == 0
        return s.value, w.value, bool(sat.value), a

    def compare(self, l: int, r: int) -> float:
        return lib().vcoh_compare(self.h, l, r)

    def job_add(self, j: int, delta):
        dl = np.ascontiguousarray(delta, np.float64)
        lib().vcoh_job_add(self.h, j, dl.ctypes.data_as(_dp))


def oracle_for(snap, queues):
    return HdrfOracle(snap, [q.hierarchy for q in queues], [q.weights for q in queues])


def tiers(drf_first: bool = True, proportion_queue_order: bool = True):
    drf = PluginOption.make("drf", EnabledHierarchy=True, EnabledQueueOrder=True, EnabledJobOrder=True)
    prop = PluginOption.make("proportion", EnabledJobEnqueued=True, EnabledQueueOrder=proportion_queue_order,
                             EnabledReclaimable=True)
    return [[drf, prop] if drf_first else [prop, drf]]


def make_pods(num, cpu, mem, pg):
    return [BuildPod("default", f"{pg}-p{i}", "", "Pending", BuildResourceList(cpu, mem), pg) for i in range(num)]


def rescaling_case() -> TestCommonStruct:
    return TestCommonStruct(
        Name="rescaling test",
        PodGroups=[BuildPodGroup("pg1", "default", "root-sci", 0, None, "Inqueue"),
                   BuildPodGroup("pg21", "default", "root-eng-dev", 0, None, "Inqueue"),
                   BuildPodGroup("pg22", "default", "root-eng-prod", 0, None, "Inqueue")],
        Pods=make_pods(10, "1", "1G", "pg1") + make_pods(10, "1", "0G", "pg21") + make_pods(10, "0", "1G", "pg22"),
        Queues=[BuildQueueWithAnnos("root-sci", 1, None, {HIER: "root/sci", WEIGHTS: "100/50"}),
                BuildQueueWithAnnos("root-eng-dev", 1, None, {HIER: "root/eng/dev", WEIGHTS: "100/50/50"}),
                BuildQueueWithAnnos("root-eng-prod", 1, None, {HIER: "root/eng/prod", WEIGHTS: "100/50/50"})],
        Nodes=[BuildNode("n", BuildResourceList("10", "10G", ("pods", "50")))],
    )


def blocking_case() -> TestCommonStruct:
    return TestCommonStruct(
        Name="blocking nodes test",
        PodGroups=[BuildPodGroup("pg1", "default", "root-pg1", 0, None, "Inqueue"),
                   BuildPodGroup("pg2", "default", "root-pg2", 0, None, "Inqueue"),
                   BuildPodGroup("pg31", "default", "root-pg3-pg31", 0, None, "Inqueue"),
                   BuildPodGroup("pg32", "default", "root-pg3-pg31", 0, None, "Inqueue"),
                   BuildPodGroup("pg4", "default", "root-pg4", 0, None, "Inqueue")],
        Pods=(make_pods(30, "1", "0G", "pg1") + make_pods(30, "1", "0G", "pg2") + make_pods(30, "1", "0G", "pg31")
              + make_pods(30, "0", "1G", "pg32") + make_pods(30, "0", "1G", "pg4")),
        Queues=[BuildQueueWithAnnos("root-pg1", 1, None, {HIER: "root/pg1", WEIGHTS: "100/25"}),
                BuildQueueWithAnnos("root-pg2", 1, None, {HIER: "root/pg2", WEIGHTS: "100/25"}),
                BuildQueueWithAnnos("root-pg3-pg31", 1, None, {HIER: "root/pg3/pg31", WEIGHTS: "100/25/50"}),
                BuildQueueWithAnnos("root-pg3-pg32", 1, None, {HIER: "root/pg3/pg32", WEIGHTS: "100/25/50"}),
                BuildQueueWithAnnos("root-pg4", 1, None, {HIER: "root/pg4", WEIGHTS: "100/25"})],
        Nodes=[BuildNode("n", BuildResourceList("30", "30G", ("pods", "500")))],
    )


def per_job_allocated(snap, decisions):
    """Resreq summed per job over the placed tasks (cpu milli, memory bytes, pods) -> {job name: vector}."""
    out = {name: np.zeros(snap.R) for name in snap.job_names}
    for d in decisions:
        t = int(d["task"])
        j = int(snap.t_job[t])
        out[snap.job_names[j]] += snap.t_resreq[:, t]
    return out


def random_tree(snap, rng, max_depth: int = 4):
    """Random hdrf annotations for the queues of a synthetic snapshot: up to `max_depth` levels below the root, shared
    nodes, root-level queues, weights < 1 / unparsable ones (clamped to 1), unequal weights. Sets the table on `snap`
    (TotalRequest = allocated at open + every pending task) and returns (hierarchy, weights) for the oracle."""
    names = ["a", "b", "c"]
    hier, wts = [], []
    for _ in range(snap.Q):
        depth = int(rng.integers(0, max_depth + 1))
        segs = ["root"] + [str(rng.choice(names)) + str(lvl) for lvl in range(depth)]
        ws = ["1"] + [str(rng.choice(["1", "2", "3", "0.5", "abc", "10", "1.5"])) for _ in range(depth)]
        hier.append("/".join(segs) if depth else "")
        wts.append("/".join(ws) if depth else "")
    from volcano_b200.synth import total_request
    snap.set_hdrf(hier, wts, total_request(snap))
    return hier, wts


def swap_queue_order(snap):
    """Put proportion's option before drf's in the configuration (the other tier order of the comparator chain)."""
    c = snap.conf
    opts = [c.plugins[i] for i in range(c.n_plugins)]
    di = next(i for i, o in enumerate(opts) if o.plugin == 3)
    pi = next(i for i, o in enumerate(opts) if o.plugin == 4)
    a, b = (c.plugins[di].plugin, c.plugins[di].enabled), (c.plugins[pi].plugin, c.plugins[pi].enabled)
    c.plugins[di].plugin, c.plugins[di].enabled = b
    c.plugins[pi].plugin, c.plugins[pi].enabled = a
