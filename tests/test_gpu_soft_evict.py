"""Preempt with PreferNoSchedule taints on the H100.

- The SOFT chain of preempt's normal reading (k_evict_rank<.., true>, k_evict_samp<true> under sampling, k_evict_pick /
  k_evict_pick_big <.., true>) launched through tools/kernels/evict_harness.cu from 1 to 200 000 nodes against a numpy
  restatement of TaintToleration's normalised score over predicateNodes and util.SortNodes' order.
- The hand-derived sessions of tests/soft_cases.py through the library.
- Random sessions of tools/fuzz_evict.make_soft_case against the CPU oracle, statement by statement."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import samp_cases as SC
from tests import samp_common as S
from tests import soft_cases as SOFT
from tests.test_gpu_samp_evict import restated
from volcano_b200 import abi

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "tools", "kernels", "_build", "evict_harness.so")
_p = C.c_void_p


class RankArgs(C.Structure):  # EhRankArgs
    _fields_ = [(n, C.c_int) for n in ("N", "R", "RT", "J", "Q", "pods_dim", "exact_sums", "n_plugins")] + \
               [(n, _p) for n in ("plugin", "tier", "enabled", "idle", "rel", "pip", "cstat", "rt_off", "rt_idx", "rt_req",
                                  "rt_flags", "rt_job", "rt_prio", "rt_evicted", "j_queue", "j_prio", "j_min", "j_ready",
                                  "q_flags", "q_over")] + \
               [(n, C.c_int) for n in ("mode", "job", "queue", "job_prio", "task_prio")] + \
               [("req", _p), ("has", C.c_uint32), ("quota_on", C.c_int), ("quota_open", C.c_int), ("qalloc_has", C.c_uint32),
                ("qdes_has", C.c_uint32), ("qalloc", _p), ("qdes", _p), ("cand", _p), ("key", _p)]


class SoftArgs(C.Structure):  # EhSoftArgs
    _fields_ = [(n, C.c_int) for n in ("w_taint", "samp", "filtered", "pct", "min_nodes", "min_pct", "start", "big")] + \
               [("seq", C.c_uint64), ("stale", C.c_uint64), ("order", _p), ("n_order", _p), ("word", _p)]


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build() compiles it")
    L = C.CDLL(LIB)
    L.eh_soft_chain.argtypes = [C.POINTER(RankArgs), C.POINTER(SoftArgs)]
    return L


def _chain_case(N, kind, rng):
    """N nodes, no running pod: a node is a candidate when it passes the static predicate and its Idle (0..3 CPUs)
    covers the preemptor's 2. Soft-taint counts 0..5 (kind "equal": 4 everywhere); "max_off_cand" puts the one maximum
    (200) on a predicate node that is not a candidate."""
    stat = rng.random(N) < 0.8
    idle = np.zeros((2, N))
    idle[0] = rng.integers(0, 4, N)
    idle[1] = 8.0
    soft = np.full(N, 4, np.uint32) if kind == "equal" else rng.integers(0, 6, N).astype(np.uint32)
    if kind == "max_off_cand":
        off = np.flatnonzero(stat & (idle[0] < 2))
        if len(off):  # the last such node: outside a sample that scans the first half of the nodes
            soft[off[-1]] = 200
    cstat = stat.astype(np.uint32) | (soft << np.uint32(8))
    return cstat, idle, soft, stat & (idle[0] >= 2)


def _expected(cstat, soft, cand, w, samp_args):
    stat = (cstat & 1).astype(bool)
    if samp_args is None:
        pred = np.flatnonzero(stat)
    else:
        pred = np.array(restated(stat.astype(np.uint8), 0, *samp_args)[0], np.int64)
    mx = int(soft[pred].max()) if len(pred) else 0
    c = soft[pred].astype(np.int64)
    sc = (np.full(len(pred), 100, np.int64) if mx == 0 else 100 - (100 * c) // mx) * w
    keep = cand[pred]
    pos = np.arange(len(pred))[keep]
    order = pred[keep][np.lexsort((pos, -sc[keep]))]  # score descending, then scan position
    return [int(n) for n in order], mx


CHAIN = [(N, kind) for N in (1, 2, 33, 1000, 25_600, 25_601, 200_000) for kind in ("random", "equal", "max_off_cand")]


@pytest.mark.parametrize("N,kind", CHAIN)
def test_soft_chain_matches_restatement(H, N, kind):
    """Every candidate handed out, in TaintToleration order over predicateNodes (every static node, or the sampled list
    with a start inside and past N), ties by scan position; the reduction word ends as (seq << 8) | max after starting
    at an earlier ranking's larger maximum. Both pick kernels where N allows the shared-memory one."""
    rng = np.random.default_rng(N * 13 + len(kind))
    cstat, idle, soft, cand = _chain_case(N, kind, rng)
    zero = np.zeros((2, N))
    keep = dict(plugin=np.array([abi.VC_PLUGIN_GANG], np.int32), tier=np.zeros(1, np.int32),
                enabled=np.array([abi.VC_EN_PREEMPTABLE], np.uint32), idle=idle, rel=zero, pip=zero, cstat=cstat,
                rt_off=np.zeros(N + 1, np.int32), j_queue=np.zeros(1, np.int32), j_prio=np.zeros(1, np.int32),
                j_min=np.zeros(1, np.int32), j_ready=np.zeros(1, np.int32), q_flags=np.zeros(1, np.uint32),
                q_over=np.zeros(1, np.uint8), req=np.array([2.0, 1.0]), cand=np.zeros(N, np.uint8),
                key=np.zeros(N, np.uint64))
    a = RankArgs(N=N, R=2, RT=0, J=1, Q=1, pods_dim=-1, exact_sums=1, n_plugins=1, mode=0, job=0, queue=0, job_prio=1,
                 task_prio=0, has=3)
    for k, v in keep.items():
        setattr(a, k, v.ctypes.data)
    seen_samp_diff = False
    for samp_args in (None, (50, 1, 5, 0), (34, 1, 5, N // 2 + 1), (5, 1, 5, 3 * N)):
        for big in ((0, 1) if N <= 25_600 else (1,)):
            if N > 30_000 and big == 1 and samp_args is not None and samp_args[0] > 10:
                continue  # one sampled drain at this size is enough (the pick at 200 000 nodes is the slow path)
            order = np.full(N, -7, np.int32)
            n_order = C.c_int32(0)
            word = C.c_uint64(0)
            seq = 5
            s = SoftArgs(w_taint=3, samp=0 if samp_args is None else 1, filtered=0, big=big, seq=seq,
                         stale=((seq - 1) << 8) | 255, order=order.ctypes.data, n_order=C.addressof(n_order),
                         word=C.addressof(word))
            if samp_args is not None:
                s.pct, s.min_nodes, s.min_pct, s.start = samp_args
            assert H.eh_soft_chain(C.byref(a), C.byref(s)) == 0
            want, mx = _expected(cstat, soft, cand, 3, samp_args)
            assert [int(x) for x in order[:n_order.value]] == want, (N, kind, samp_args, big)
            assert word.value == (seq << 8) | mx, (N, kind, samp_args, big, word.value, mx)
            if samp_args is not None and mx != _expected(cstat, soft, cand, 3, None)[1]:
                seen_samp_diff = True
    if N >= 1000 and kind == "max_off_cand":
        assert seen_samp_diff  # a maximum outside the sample occurred


def _gpu(snap):
    from volcano_b200 import engine
    engine.init(0)
    return engine.gpu_engine(snap)


@pytest.mark.parametrize("case", sorted(SOFT.CASES))
def test_hand_derived_cases(case):
    snap, want = SOFT.CASES[case]()
    assert SC.statements(snap, _gpu(snap).preempt) == want


def test_sessions_match_the_oracle():
    """320 random sessions of make_soft_case: allocate placements, preempt / reclaim statements and visits, and under
    sampling the index, identical to the oracle. Not vacuous: sessions with soft taints where the oracle's preempt
    statements change when tainttoleration.weight drops to 0, under sampling and without."""
    from tools.fuzz_evict import make_soft_case
    checked, changed, evictions = 0, {True: 0, False: 0}, 0
    for seed in range(320):
        tc, tiers, actions, conf = make_soft_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = S.run(snap)
        res = _gpu(snap)
        assert S.same(res, ref), (seed, actions, conf)
        checked += 1
        evictions += sum(len(getattr(ref, a).decisions) for a in ("preempt", "reclaim") if getattr(ref, a) is not None)
        if snap.conf.w_taint_toleration and ref.preempt is not None and len(ref.preempt.decisions):
            for t in tiers:
                for o in t:
                    if o.name == "nodeorder":
                        o.arguments["tainttoleration.weight"] = 0
            flat = S.run(tc.RegisterSession(tiers, actions=actions, **conf))
            if flat.preempt is None or not S.same(ref, flat, index=False):
                changed["percentage_nodes_to_find" in conf] += 1
    assert checked >= 250 and evictions > 0
    assert changed[True] >= 3 and changed[False] >= 3, changed
