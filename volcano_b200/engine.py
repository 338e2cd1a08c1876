"""ctypes binding of libvcalloc.so — the product path. There is no CPU fallback: if the CUDA
library is missing or no device is present, constructing an Engine raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Tuple

import numpy as np

from . import abi
from .snapshot import Snapshot
from .uthelper import AllocateResult

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libvcalloc.so")
_lib: Optional[C.CDLL] = None

DECISION_DTYPE = np.dtype([("task", "<i4"), ("node", "<i4"), ("kind", "<i4"), ("visit", "<i4"), ("score", "<f8")])
VISIT_DTYPE = np.dtype([("job", "<i4"), ("outcome", "<i4"), ("first_op", "<i4"), ("n_ops", "<i4")])

_dp, _i32p, _u64p, _i64p = (C.POINTER(t) for t in (C.c_double, C.c_int32, C.c_uint64, C.c_int64))


class VcError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libvcalloc error {code}: {msg}")
        self.code = code


def load_library() -> C.CDLL:
    """dlopen the in-tree library; raises (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise FileNotFoundError(f"{_LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _lib = abi.bind(C.CDLL(_LIB_PATH))
    return _lib


def _check(rc: int):
    if rc != 0:
        raise VcError(rc, load_library().vc_last_error().decode())


def init(device: int = 0):
    _check(load_library().vc_init(device))


def debug_option(name: str, value: int):
    """Diagnostic switch by its environment-variable name (kernel instance selection, timers); results never change."""
    _check(load_library().vc_debug_option(name.encode(), int(value)))


def _struct_array(ptr, n, dtype):
    if n == 0:
        return np.zeros(0, dtype)
    buf = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), (n * dtype.itemsize,))
    return buf.view(dtype).copy()


class Engine:
    """One scheduling session on one GPU: upload -> allocate / dense pass."""

    def __init__(self, snap: Snapshot, device: int = 0):
        self.L = load_library()
        init(device)
        self.snap = snap
        self.h = C.c_void_p()
        d = snap.dims()
        _check(self.L.vc_snapshot_create(C.byref(d), C.byref(self.h)))
        self._uploaded = False

    def close(self):
        if getattr(self, "h", None):
            self.L.vc_snapshot_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, snap: Optional[Snapshot] = None):
        if snap is not None:
            self.snap = snap
        s = self.snap
        n, t, c, j, q = s.nodes(), s.tasks(), s.classes(), s.jobs(), s.queues()
        topo = s.topology()
        if topo is not None:
            _check(self.L.vc_snapshot_set_topology(self.h, C.byref(topo)))
        hd = s.hdrf()  # drf's enableHierarchy: restated on every upload, None clears it
        _check(self.L.vc_snapshot_set_hdrf(self.h, C.byref(hd) if hd is not None else None))
        bt = s.backfill_tasks()  # the list stays in effect until replaced: always (re)state it, an empty one clears it
        _check(self.L.vc_snapshot_set_backfill(self.h, s.B, C.byref(bt) if bt is not None else None))
        rt = s.running_tasks()  # node.Tasks (victim candidates of preempt / reclaim) + per-task flags; restated on every upload
        tf = s.t_flags.ctypes.data_as(C.POINTER(C.c_uint32)) if s.T else None
        _check(self.L.vc_snapshot_set_running(self.h, C.byref(rt) if rt is not None else None, tf))
        po = s.preempt_options()  # the preempt action's arguments; restated on every upload, None restores the defaults
        _check(self.L.vc_snapshot_set_preempt_options(self.h, C.byref(po) if po is not None else None))
        vg = s.victim_guards()  # the pdb / cdp votes' table; restated on every upload, None clears it
        _check(self.L.vc_snapshot_set_victim_guards(self.h, C.byref(vg) if vg is not None else None))
        nom = getattr(s, "t_nominated", None)  # Pod.Status.NominatedNodeName per pending task; restated on every upload
        has_nom = nom is not None and s.T and bool((nom >= 0).any())
        _check(self.L.vc_snapshot_set_nominated(self.h, nom.ctypes.data_as(C.POINTER(C.c_int32)) if has_nom else None))
        _check(self.L.vc_snapshot_upload(self.h, C.byref(n), C.byref(t), C.byref(c), C.byref(j), C.byref(q),
                                         C.byref(s.conf)))
        self._uploaded = True

    def update_nodes(self, idx, idle, used, releasing, pipelined, k8s_requested, k8s_nonzero_requested, pod_count):
        """Incremental upload of the accounting rows of the nodes `idx` (arrays compact: [dim][len(idx)])."""
        idx = np.ascontiguousarray(idx, np.int32)
        arrs = [np.ascontiguousarray(a, np.float64) for a in (idle, used, releasing, pipelined, k8s_requested, k8s_nonzero_requested)]
        pods = np.ascontiguousarray(pod_count, np.int32)
        rows = abi.vc_nodes()
        rows.idle, rows.used, rows.releasing, rows.pipelined = (a.ctypes.data_as(_dp) for a in arrs[:4])
        rows.k8s_requested, rows.k8s_nonzero_requested = arrs[4].ctypes.data_as(_dp), arrs[5].ctypes.data_as(_dp)
        rows.pod_count = pods.ctypes.data_as(_i32p)
        _check(self.L.vc_snapshot_update_nodes(self.h, len(idx), idx.ctypes.data_as(_i32p), C.byref(rows)))

    def allocate(self) -> AllocateResult:
        if not self._uploaded:
            self.upload()
        r = C.c_void_p()
        _check(self.L.vc_allocate_run(self.h, C.byref(r)))
        return self._result(r)

    def backfill(self) -> AllocateResult:
        """The backfill action on the session state allocate() left (decision.task indexes snap.backfill_task_keys)."""
        if not self._uploaded:
            self.upload()
        r = C.c_void_p()
        _check(self.L.vc_backfill_run(self.h, C.byref(r)))
        return self._result(r)

    def preempt(self) -> AllocateResult:
        """The preempt action on the session state the preceding actions left (VC_OP_EVICT: task indexes
        snap.running_task_keys)."""
        if not self._uploaded:
            self.upload()
        r = C.c_void_p()
        _check(self.L.vc_preempt_run(self.h, C.byref(r)))
        return self._result(r)

    def reclaim(self) -> AllocateResult:
        if not self._uploaded:
            self.upload()
        r = C.c_void_p()
        _check(self.L.vc_reclaim_run(self.h, C.byref(r)))
        return self._result(r)

    def _result(self, r) -> AllocateResult:
        try:
            nd = self.L.vc_result_num_decisions(r)
            nv = self.L.vc_result_num_visits(r)
            nf = self.L.vc_result_num_fit_errors(r)
            dec = _struct_array(self.L.vc_result_decisions(r), nd, DECISION_DTYPE)
            vis = _struct_array(self.L.vc_result_visits(r), nv, VISIT_DTYPE)
            fe = np.ctypeslib.as_array(self.L.vc_result_fit_errors(r), (nf,)).copy() if nf else np.zeros(0, np.int32)
            nj = C.c_size_t(0)
            ja = self.L.vc_result_job_allocated_hypernodes(r, C.byref(nj))
            job_alloc = np.ctypeslib.as_array(ja, (nj.value,)).copy() if nj.value else None
            st = self.L.vc_result_stats(r).contents
            stats = {k: (list(getattr(st, k)) if k in ("prof_cycles", "group_reentry") else getattr(st, k)) for k, _ in abi.vc_stats._fields_}
        finally:
            self.L.vc_result_free(r)
        res = AllocateResult(dec, vis, fe, stats)
        res.job_allocated_hypernodes = job_alloc
        return res

    # one session across the GPUs of a node (SURVEY §8e): see include/vcalloc.h vc_comm_*
    def comm_create(self, world: int, rank: int) -> bytes:
        buf = (C.c_ubyte * abi.VC_COMM_HANDLE_BYTES)()
        _check(self.L.vc_comm_create(self.h, world, rank, buf))
        self._uploaded = False
        return bytes(buf)

    def comm_attach(self, handles: bytes):
        _check(self.L.vc_comm_attach(self.h, handles))

    def comm_prepare(self):
        _check(self.L.vc_comm_prepare(self.h))

    def set_shard(self, begin: int, end: int):
        _check(self.L.vc_snapshot_set_shard(self.h, begin, end))

    def score_matrix(self, want_mask=True, want_score=True):
        if not self._uploaded:
            self.upload()
        s = self.snap
        mw = (s.N + 63) // 64
        mask = np.zeros((s.T, mw), np.uint64) if want_mask else None
        score = np.zeros((s.T, s.N), np.float64) if want_score else None
        bs = np.zeros(s.T, np.float64)
        bn = np.zeros(s.T, np.int32)
        _check(self.L.vc_score_matrix(self.h, mask.ctypes.data_as(_u64p) if want_mask else None,
                                      score.ctypes.data_as(_dp) if want_score else None,
                                      bs.ctypes.data_as(_dp), bn.ctypes.data_as(_i32p)))
        return mask, score, bs, bn

    def score_matrix_device(self, repeats: int = 3) -> Tuple[float, float, int]:
        """-> (ms per dense pass, ms of the materialising kernel alone, algorithmic bytes)."""
        if not self._uploaded:
            self.upload()
        ms = (C.c_double * 2)()
        nbytes = C.c_int64()
        _check(self.L.vc_score_matrix_device(self.h, repeats, ms, C.byref(nbytes)))
        return ms[0], ms[1], nbytes.value

    def queue_deserved(self):
        s = self.snap
        des = np.zeros((s.R, s.Q))
        share = np.zeros(s.Q)
        _check(self.L.vc_queue_deserved(self.h, des.ctypes.data_as(_dp), share.ctypes.data_as(_dp)))
        return des, share

    # node-sharded dense pass building blocks (device pointers for torch.distributed)
    def dense_begin(self):
        _check(self.L.vc_dense_begin(self.h))

    def dense_stats_ptr(self) -> Tuple[int, int]:
        p, n = _i32p(), C.c_int32()
        _check(self.L.vc_dense_stats(self.h, C.byref(p), C.byref(n)))
        return C.cast(p, C.c_void_p).value, n.value

    def dense_finish(self, materialize: bool):
        _check(self.L.vc_dense_finish(self.h, 1 if materialize else 0))

    def dense_best_ptrs(self) -> Tuple[int, int]:
        ps, pn = _dp(), _i32p()
        _check(self.L.vc_dense_best(self.h, C.byref(ps), C.byref(pn)))
        return C.cast(ps, C.c_void_p).value, C.cast(pn, C.c_void_p).value


def gpu_engine(snap: Snapshot, device: int = 0) -> AllocateResult:
    """Snapshot -> AllocateResult on the GPU (the `engine` callable for uthelper.TestCommonStruct.Run)."""
    e = Engine(snap, device)
    try:
        e.upload()
        actions = [a for a in snap.actions if a != "enqueue"]  # the configured action list, scheduler.go:124-153
        if "allocate" in actions or not any(a in ("preempt", "reclaim") for a in actions):
            res = e.allocate()
        else:  # an action list without allocate (the reference's preempt / reclaim unit tests)
            res = AllocateResult(np.zeros(0, DECISION_DTYPE), np.zeros(0, VISIT_DTYPE), np.zeros(0, np.int32))
        for a in actions:
            if a == "backfill" and snap.B > 0:
                res.backfill = e.backfill()
            elif a == "preempt":
                res.preempt = e.preempt()
            elif a == "reclaim":
                res.reclaim = e.reclaim()
        return res
    finally:
        e.close()
