"""Preempt and reclaim under feasible-node sampling: the loader of the oracle extension
(tools/samp_evict_oracle/samp_evict_oracle.cpp), an engine callable over it, and the PredicateNodes log it keeps."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from volcano_b200 import abi
from volcano_b200.uthelper import AllocateResult

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = os.path.join(ROOT, "tools", "samp_evict_oracle", "_build", "libsamp_evict_oracle.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        import __graft_entry__
        from oracle import pyoracle
        __graft_entry__.build_samp_evict_oracle()
        L = C.CDLL(_LIB)
        ref = pyoracle.lib()
        for name in ("vco_session_create", "vco_session_destroy", "vco_session_set_running", "vco_allocate_run",
                     "vco_reclaim", "vco_num_decisions", "vco_num_visits", "vco_num_fit_errors", "vco_decisions",
                     "vco_visits", "vco_fit_errors", "vco_last_processed_node_index"):
            getattr(L, name).restype = getattr(ref, name).restype
            getattr(L, name).argtypes = getattr(ref, name).argtypes
        L.vcot_set_preempt_options.argtypes = [C.c_void_p, C.POINTER(abi.vc_preempt_options)]
        L.vcot_preempt.argtypes = [C.c_void_p]
        for name in ("vcse_allocate", "vcse_preempt", "vcse_reclaim"):
            getattr(L, name).argtypes = [C.c_void_p]
        L.vcse_index.restype = C.c_int64
        L.vcse_index.argtypes = [C.c_void_p]
        L.vcse_node_errors.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
        L.vcse_calls.restype = C.c_int64
        L.vcse_calls.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int64]
        L.vcse_forget.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class SampOracle:
    """A CPU oracle session whose preempt / reclaim follow the sampling contract (and the preempt options of the
    snapshot). `restated=False` runs the unchanged oracle's actions instead (allocate, preempt, reclaim) for comparison."""

    def __init__(self, snap, restated: bool = True):
        L = lib()
        self.snap, self.restated = snap, restated
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
            lib().vcse_forget(self.h)
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
            raise RuntimeError(f"sampling oracle {what} rc={rc}")
        from oracle.pyoracle import DECISION_DTYPE, VISIT_DTYPE
        L = lib()
        nd, nv, nf = L.vco_num_decisions(self.h), L.vco_num_visits(self.h), L.vco_num_fit_errors(self.h)
        dec = np.ctypeslib.as_array(C.cast(L.vco_decisions(self.h), C.POINTER(C.c_uint8)), (nd * DECISION_DTYPE.itemsize,)
                                    ).view(DECISION_DTYPE).copy() if nd else np.zeros(0, DECISION_DTYPE)
        vis = np.ctypeslib.as_array(C.cast(L.vco_visits(self.h), C.POINTER(C.c_uint8)), (nv * VISIT_DTYPE.itemsize,)
                                    ).view(VISIT_DTYPE).copy() if nv else np.zeros(0, VISIT_DTYPE)
        fe = np.ctypeslib.as_array(L.vco_fit_errors(self.h), (nf,)).copy() if nf else np.zeros(0, np.int32)
        return AllocateResult(dec, vis, fe, {"last_processed_node_index": int(L.vcse_index(self.h))})

    def allocate(self):
        return self._run(lib().vcse_allocate if self.restated else lib().vco_allocate_run, "allocate")

    def preempt(self):
        return self._run(lib().vcse_preempt if self.restated else lib().vcot_preempt, "preempt")

    def reclaim(self):
        return self._run(lib().vcse_reclaim if self.restated else lib().vco_reclaim, "reclaim")

    def node_errors(self) -> np.ndarray:
        out = np.zeros(max(self.snap.T, 1), np.uint8)
        lib().vcse_node_errors(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)))
        return out[:self.snap.T]

    def calls(self):
        """Every PredicateNodes call of the evicting actions so far: dicts of task, P (length of the scanned list),
        processed, index (after the call) and nodes (predicateNodes in scan order)."""
        L = lib()
        n = L.vcse_calls(self.h, None, 0)
        buf = np.zeros(max(n, 1), np.int32)
        L.vcse_calls(self.h, buf.ctypes.data_as(C.POINTER(C.c_int32)), n)
        out, i = [], 0
        while i < n:
            t, P, proc, idx, m = (int(x) for x in buf[i:i + 5])
            out.append({"task": t, "P": P, "processed": proc, "index": idx, "nodes": [int(x) for x in buf[i + 5:i + 5 + m]]})
            i += 5 + m
        return out


def run(snap, restated: bool = True, keep=None) -> AllocateResult:
    """Snapshot -> AllocateResult through the oracle, the configured actions in order. keep(oracle) is called before
    the session closes."""
    o = SampOracle(snap, restated)
    try:
        actions = [a for a in snap.actions if a != "enqueue"]
        if "allocate" in actions:
            res = o.allocate()
        else:
            from oracle.pyoracle import DECISION_DTYPE, VISIT_DTYPE
            res = AllocateResult(np.zeros(0, DECISION_DTYPE), np.zeros(0, VISIT_DTYPE), np.zeros(0, np.int32))
        for a in actions:
            if a == "preempt":
                res.preempt = o.preempt()
            elif a == "reclaim":
                res.reclaim = o.reclaim()
        if keep is not None:
            keep(o)
        return res
    finally:
        o.close()


def same(a: AllocateResult, b: AllocateResult, index: bool = True) -> bool:
    """Identical allocate placements and identical statements and visits of preempt and reclaim; with `index`, the
    same lastProcessedNodeIndex after each evicting action."""
    for name in ("preempt", "reclaim"):
        x, y = getattr(a, name), getattr(b, name)
        if (x is None) != (y is None):
            return False
        if x is None:
            continue
        if not (np.array_equal(x.visits, y.visits) and all(np.array_equal(x.decisions[f], y.decisions[f])
                                                            for f in ("task", "node", "kind", "visit"))):
            return False
        if index and x.stats["last_processed_node_index"] != y.stats["last_processed_node_index"]:
            return False
    return np.array_equal(a.decisions["task"], b.decisions["task"]) and np.array_equal(a.decisions["node"], b.decisions["node"])
