"""The pdb and cdp victim votes: the loader of the oracle extension (tools/guard_oracle/guard_oracle.cpp) and an engine
callable over it that runs the configured actions with the session's victim-guard table."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from tests import samp_common as S
from volcano_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = os.path.join(ROOT, "tools", "guard_oracle", "_build", "libguard_oracle.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        import __graft_entry__
        from oracle import pyoracle
        __graft_entry__.build_guard_oracle()
        L = C.CDLL(_LIB)
        ref = pyoracle.lib()
        for name in ("vco_session_create", "vco_session_destroy", "vco_session_set_running", "vco_allocate_run",
                     "vco_num_decisions", "vco_num_visits", "vco_num_fit_errors", "vco_decisions", "vco_visits",
                     "vco_fit_errors"):
            getattr(L, name).restype = getattr(ref, name).restype
            getattr(L, name).argtypes = getattr(ref, name).argtypes
        L.vcot_set_preempt_options.argtypes = [C.c_void_p, C.POINTER(abi.vc_preempt_options)]
        L.vcgo_set_victim_guards.argtypes = [C.c_void_p, C.POINTER(abi.vc_victim_guards)]
        for name in ("vcse_allocate", "vcgo_preempt", "vcgo_reclaim"):
            getattr(L, name).argtypes = [C.c_void_p]
        L.vcse_index.restype = C.c_int64
        L.vcse_index.argtypes = [C.c_void_p]
        L.vcgo_vote.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_uint8)]
        L.vcgo_forget.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class GuardOracle(S.SampOracle):
    """A sampling-oracle session whose preempt / reclaim add the pdb and cdp votes (the snapshot's victim guards)."""

    def __init__(self, snap):
        L = lib()
        self.snap, self.restated = snap, True
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
            raise RuntimeError(f"guard oracle {what} rc={rc}")
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
        return self._run(lib().vcgo_preempt, "preempt")

    def reclaim(self):
        return self._run(lib().vcgo_reclaim, "reclaim")

    def vote(self, plugin: int, rts) -> list:
        """One plugin's answer on the running tasks `rts` (in that order): the running-task indices it returns."""
        a = np.array(rts, np.int32)
        out = np.zeros(max(len(a), 1), np.uint8)
        lib().vcgo_vote(self.h, plugin, a.ctypes.data_as(C.POINTER(C.c_int32)), len(a), out.ctypes.data_as(C.POINTER(C.c_uint8)))
        return [int(r) for r, y in zip(a, out) if y]


def run(snap):
    """Snapshot -> AllocateResult through the guard oracle, the configured actions in order."""
    o = GuardOracle(snap)
    try:
        from oracle.pyoracle import DECISION_DTYPE, VISIT_DTYPE
        from volcano_b200.uthelper import AllocateResult
        actions = [a for a in snap.actions if a != "enqueue"]
        res = o.allocate() if "allocate" in actions else AllocateResult(np.zeros(0, DECISION_DTYPE),
                                                                          np.zeros(0, VISIT_DTYPE), np.zeros(0, np.int32))
        for a in actions:
            if a == "preempt":
                res.preempt = o.preempt()
            elif a == "reclaim":
                res.reclaim = o.reclaim()
        return res
    finally:
        o.close()


def evicted(snap, res) -> list:
    """Pod keys of the Evict operations of committed statements, preempt then reclaim."""
    out = []
    for name in ("preempt", "reclaim"):
        ar = getattr(res, name, None)
        if ar is None:
            continue
        for v in ar.visits:
            if v["outcome"] == abi.VC_VISIT_COMMIT:
                for op in ar.decisions[v["first_op"]: v["first_op"] + v["n_ops"]]:
                    if op["kind"] == abi.VC_OP_EVICT:
                        out.append(snap.running_task_keys[op["task"]])
    return out
