"""Preempt and reclaim with the network-topology-aware plugin: the loader of the oracle extension
(tools/nta_evict_oracle/nta_evict_oracle.cpp) and an engine callable over it that runs the configured actions on the
session's HyperNode tree, victim guards and preempt options."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from tests import guard_common as G
from volcano_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = os.path.join(ROOT, "tools", "nta_evict_oracle", "_build", "libnta_evict_oracle.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        import __graft_entry__
        from oracle import pyoracle
        __graft_entry__.build_nta_evict_oracle()
        L = C.CDLL(_LIB)
        ref = pyoracle.lib()
        for name in ("vco_session_create", "vco_session_destroy", "vco_session_set_running", "vco_allocate_run",
                     "vco_num_decisions", "vco_num_visits", "vco_num_fit_errors", "vco_decisions", "vco_visits",
                     "vco_fit_errors", "vco_session_set_topology", "vco_hypernode_status"):
            getattr(L, name).restype = getattr(ref, name).restype
            getattr(L, name).argtypes = getattr(ref, name).argtypes
        L.vcot_set_preempt_options.argtypes = [C.c_void_p, C.POINTER(abi.vc_preempt_options)]
        L.vcgo_set_victim_guards.argtypes = [C.c_void_p, C.POINTER(abi.vc_victim_guards)]
        for name in ("vcse_allocate", "vcnta_preempt", "vcnta_reclaim"):
            getattr(L, name).argtypes = [C.c_void_p]
        L.vcse_index.restype = C.c_int64
        L.vcse_index.argtypes = [C.c_void_p]
        L.vcgo_forget.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class NtaOracle(G.GuardOracle):
    """A guard-oracle session on the snapshot's HyperNode tree whose preempt / reclaim accept the network-topology-aware
    plugin and soft-mode topology jobs."""

    def __init__(self, snap):
        L = lib()
        self.snap, self.restated = snap, True
        d, n, t, c, j, q = snap.dims(), snap.nodes(), snap.tasks(), snap.classes(), snap.jobs(), snap.queues()
        self.h = L.vco_session_create(C.byref(d), C.byref(n), C.byref(t), C.byref(c), C.byref(j), C.byref(q),
                                      C.byref(snap.conf), 1)
        assert self.h
        topo = snap.topology()
        if topo is not None:
            L.vco_session_set_topology(self.h, C.byref(topo))
        rt = snap.running_tasks()
        if rt is not None or snap.t_flags.any():
            tf = snap.t_flags.ctypes.data_as(C.POINTER(C.c_uint32)) if snap.T else None
            assert L.vco_session_set_running(self.h, C.byref(rt) if rt is not None else None, tf) == 0
        po = snap.preempt_options()
        assert L.vcot_set_preempt_options(self.h, C.byref(po) if po is not None else None) == 0
        vg = snap.victim_guards()
        assert L.vcgo_set_victim_guards(self.h, C.byref(vg) if vg is not None else None) == 0

    def close(self):
        if self.h:
            lib().vcgo_forget(self.h)
            lib().vco_session_destroy(self.h)
            self.h = None

    def _run(self, fn, what):
        rc = fn(self.h)
        if rc != 0:
            raise RuntimeError(f"nta evict oracle {what} rc={rc}")
        from oracle.pyoracle import DECISION_DTYPE, VISIT_DTYPE
        from volcano_b200.uthelper import AllocateResult
        L = lib()
        nd, nv, nf = L.vco_num_decisions(self.h), L.vco_num_visits(self.h), L.vco_num_fit_errors(self.h)
        dec = np.ctypeslib.as_array(C.cast(L.vco_decisions(self.h), C.POINTER(C.c_uint8)), (nd * DECISION_DTYPE.itemsize,)
                                    ).view(DECISION_DTYPE).copy() if nd else np.zeros(0, DECISION_DTYPE)
        vis = np.ctypeslib.as_array(C.cast(L.vco_visits(self.h), C.POINTER(C.c_uint8)), (nv * VISIT_DTYPE.itemsize,)
                                    ).view(VISIT_DTYPE).copy() if nv else np.zeros(0, VISIT_DTYPE)
        fe = np.ctypeslib.as_array(L.vco_fit_errors(self.h), (nf,)).copy() if nf else np.zeros(0, np.int32)
        return AllocateResult(dec, vis, fe, {"last_processed_node_index": int(L.vcse_index(self.h))})

    def allocate(self):
        return self._run(lib().vcse_allocate, "allocate")

    def preempt(self):
        return self._run(lib().vcnta_preempt, "preempt")

    def reclaim(self):
        return self._run(lib().vcnta_reclaim, "reclaim")

    def hn_used(self, h: int) -> np.ndarray:
        """hyperNodeResourceCache[h].used as the session stands, per resource dimension."""
        used = np.zeros(abi.VC_MAX_DIMS, np.float64)
        alloc = np.zeros(abi.VC_MAX_DIMS, np.float64)
        lib().vco_hypernode_status(self.h, h, alloc.ctypes.data_as(C.POINTER(C.c_double)),
                                   used.ctypes.data_as(C.POINTER(C.c_double)))
        return used[: self.snap.R].copy()


def run(snap, keep=None):
    """Snapshot -> AllocateResult through the oracle, the configured actions in order. `keep`, a list, receives
    hyperNodeResourceCache.used of every hypernode after each action, as (action, [H][R] array)."""
    from oracle.pyoracle import DECISION_DTYPE, VISIT_DTYPE
    from volcano_b200.uthelper import AllocateResult
    o = NtaOracle(snap)
    try:
        actions = [a for a in snap.actions if a != "enqueue"]
        res = o.allocate() if "allocate" in actions else AllocateResult(np.zeros(0, DECISION_DTYPE),
                                                                          np.zeros(0, VISIT_DTYPE), np.zeros(0, np.int32))
        H = len(snap.hn_names) if snap.hn_member is not None else 1
        for a in actions:
            if a == "preempt":
                res.preempt = o.preempt()
            elif a == "reclaim":
                res.reclaim = o.reclaim()
            if keep is not None:
                keep.append((a, np.array([o.hn_used(h) for h in range(H)])))
        return res
    finally:
        o.close()


def evict_changed(a, b) -> bool:
    """The same allocate placements, and different preempt / reclaim statements or visits: the difference comes from
    the evicting actions themselves."""
    from tests import samp_common as S
    same_alloc = np.array_equal(a.decisions["task"], b.decisions["task"]) and np.array_equal(a.decisions["node"], b.decisions["node"])
    return bool(same_alloc and not S.same(a, b, index=False))
