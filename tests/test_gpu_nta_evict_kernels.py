"""The network-topology-aware instances of the preempt / reclaim kernels on the H100, through tools/kernels/evict_harness.cu,
against a numpy restatement of hn_binpack_score / nta_node_score / total_score / util.SortNodes in the device's operation
order (bit for bit):
- k_evict_rank<16, 8 | VC_MAX_DIMS, false, false, true>: the candidates' keys, 1 to 200 000 nodes, 1 to 3 tier levels,
  nodes outside any hypernode of a level, hypernodes at and over their allocatable (score 0);
- the SOFT+NTA chain (k_evict_rank<.., true, false, true>, k_evict_samp<true>, k_evict_pick / k_evict_pick_big
  <SAMP, true, true>): the stored term and the order of every hand-out;
- k_evict_apply<true>: hyperNodeResourceCache.used after a statement and after its undo, and back at its bits for
  integer-valued requests."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.test_gpu_evict_kernels import ApplyArgs
from tests.test_gpu_samp_evict import restated
from tests.test_gpu_soft_evict import RankArgs, SoftArgs
from volcano_b200 import abi

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "tools", "kernels", "_build", "evict_harness.so")
_p = C.c_void_p


class NtaArgs(C.Structure):  # EhNtaArgs
    _fields_ = [("L", C.c_int), ("H", C.c_int), ("weight", C.c_int)] + \
               [(n, _p) for n in ("member", "hn_alloc", "hn_used", "tier_w", "dim_weight", "nta_term")]


class NtaApply(C.Structure):  # EhNtaApply
    _fields_ = [("L", C.c_int), ("H", C.c_int), ("member", _p), ("hn_used", _p), ("rt_has", _p), ("has", C.c_uint32)]


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build() compiles it")
    L = C.CDLL(LIB)
    L.eh_nta_rank.argtypes = [C.POINTER(RankArgs), C.POINTER(NtaArgs)]
    L.eh_nta_soft_chain.argtypes = [C.POINTER(RankArgs), C.POINTER(SoftArgs), C.POINTER(NtaArgs)]
    L.eh_apply_nta.argtypes = [C.POINTER(ApplyArgs), C.POINTER(NtaApply)]
    return L


def _tree(N, L, R, rng):
    """member [L][N] over hypernodes numbered level by level (about N/8, N/64, then 1 per level; 15 % of the nodes in none
    of a level's), integral allocatable and non-integer used [R][H]."""
    sizes = [max(1, N // 8), max(1, N // 64), 1][:L]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    Hn = int(off[-1])
    member = np.empty((L, N), np.int32)
    for l in range(L):
        m = off[l] + rng.integers(0, sizes[l], N)
        member[l] = np.where(rng.random(N) < 0.15, -1, m)
    alloc = rng.integers(16, 65, (R, Hn)).astype(np.float64)
    used = alloc * rng.uniform(0.0, 0.9, (R, Hn))
    return member, alloc, used


def _preemptor(R, rng):
    req = np.zeros(R)
    req[0], req[1] = 2.0, 1.5
    has = 3
    for d in range(2, R):
        if rng.random() < 0.6:
            has |= 1 << d
            req[d] = rng.choice([0.05, 1.0, 2.5])  # 0.05: below MinResource, not weighed
    dw = np.array([5, 1] + [int(rng.choice([-1, 0, 2])) for _ in range(2, R)], np.int32)
    return req, has, dw


def _edge(alloc, used, req, has, rng):
    """a third of the hypernodes at allocatable (used + request == allocatable on every weighed dim), a sixth over it"""
    Hn = alloc.shape[1]
    kind = rng.random(Hn)
    for h in range(Hn):
        if kind[h] < 1 / 3:
            for d in range(alloc.shape[0]):
                used[d, h] = alloc[d, h] - req[d]
        elif kind[h] < 0.5:
            used[0, h] = alloc[0, h] - req[0] + 0.5
    return kind


def _hn_scores(req, has, dw, alloc, used):
    out = []
    for h in range(alloc.shape[1]):
        total, tw, zero = 0.0, 0, False
        for d in range(len(req)):
            rq = float(req[d])
            if d >= 2 and not (has >> d) & 1:
                continue
            if not rq >= 0.1:
                continue
            w = int(dw[d])
            if w < 0:
                continue
            al, u = float(alloc[d, h]), float(used[d, h])
            if u + rq > al:
                zero = True
                break
            total += float(w) * ((u + rq) / al)
            tw += w
        out.append(0.0 if zero or tw <= 0 else total / float(tw))
    return np.array(out)


def _terms(member, hs, tier_w, weight):
    total = np.zeros(member.shape[1])
    for l in range(member.shape[0]):
        ts = np.where(member[l] < 0, 1.0, hs[np.maximum(member[l], 0)])
        total = total + tier_w[l] * ts
    tw = 0.0
    for w in tier_w:
        tw += w
    return 100.0 * float(weight) * (total / tw)


def _key(x):
    u = np.ascontiguousarray(x, np.float64).view(np.uint64)
    return np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))


def _rank_inputs(N, R, rng, req, has, cstat):
    """no running pod: a node is a candidate when it passes the static predicate and its Idle CPUs (0..3) cover 2"""
    idle = np.full((R, N), 1e6)
    idle[0] = rng.integers(0, 4, N)
    zero = np.zeros((R, N))
    keep = dict(plugin=np.array([abi.VC_PLUGIN_GANG], np.int32), tier=np.zeros(1, np.int32),
                enabled=np.array([abi.VC_EN_PREEMPTABLE], np.uint32), idle=idle, rel=zero, pip=zero, cstat=cstat,
                rt_off=np.zeros(N + 1, np.int32), j_queue=np.zeros(1, np.int32), j_prio=np.zeros(1, np.int32),
                j_min=np.zeros(1, np.int32), j_ready=np.zeros(1, np.int32), q_flags=np.zeros(1, np.uint32),
                q_over=np.zeros(1, np.uint8), req=req, cand=np.zeros(N, np.uint8), key=np.zeros(N, np.uint64))
    a = RankArgs(N=N, R=R, RT=0, J=1, Q=1, pods_dim=-1, exact_sums=1, n_plugins=1, mode=0, job=0, queue=0, job_prio=1,
                 task_prio=0, has=has)
    for k, v in keep.items():
        setattr(a, k, v.ctypes.data)
    cand = ((cstat & 1) != 0) & (idle[0] >= 2)
    return a, keep, cand


def _nta_args(member, alloc, used, tier_w, dw, weight, term_out):
    x = NtaArgs(L=member.shape[0], H=alloc.shape[1], weight=weight)
    keep = dict(member=np.ascontiguousarray(member), hn_alloc=np.ascontiguousarray(alloc),
                hn_used=np.ascontiguousarray(used), tier_w=np.asarray(tier_w, np.float64), dim_weight=dw, nta_term=term_out)
    for k, v in keep.items():
        setattr(x, k, v.ctypes.data)
    return x, keep


TIER_W = [1.0, 0.8, 0.8 * 0.8]
RANK = [(N, L, R) for N in (1, 2, 33, 1000, 25_600, 25_601, 200_000) for L in (1, 2, 3) for R in (2, 10)]


@pytest.mark.parametrize("N,L,R", RANK)
def test_nta_rank_keys_vs_numpy(H, N, L, R):
    rng = np.random.default_rng(N * 31 + L * 7 + R)
    member, alloc, used = _tree(N, L, R, rng)
    req, has, dw = _preemptor(R, rng)
    kind = _edge(alloc, used, req, has, rng)
    cstat = (rng.random(N) < 0.8).astype(np.uint32)
    a, keep, cand = _rank_inputs(N, R, rng, req, has, cstat)
    term_out = np.full(N, -7.0)
    x, keep2 = _nta_args(member, alloc, used, TIER_W[:L], dw, 10, term_out)
    assert H.eh_nta_rank(C.byref(a), C.byref(x)) == 0
    hs = _hn_scores(req, has, dw, alloc, used)
    term = _terms(member, hs, TIER_W[:L], 10)
    got_cand = keep["cand"]
    assert np.array_equal(got_cand.astype(bool), cand), (N, L, R)
    want = np.where(cand, _key(0.0 + (0.0 + term)), np.uint64(0))
    assert np.array_equal(keep["key"], want), (N, L, R)
    assert np.all(term_out == 0.0)  # without SOFT the term is in the key only
    if N >= 1000:  # the edges the case is built for are there
        assert (hs == 0.0).any() and (kind < 1 / 3).any() and (member < 0).any()
        assert len(np.unique(keep["key"][cand])) > 10


def _chain_expected(cstat, soft, cand, term, w, samp_args):
    stat = (cstat & 1).astype(bool)
    if samp_args is None:
        pred = np.flatnonzero(stat)
    else:
        pred = np.array(restated(stat.astype(np.uint8), 0, *samp_args)[0], np.int64)
    mx = int(soft[pred].max()) if len(pred) else 0
    c = soft[pred].astype(np.int64)
    sc = (np.full(len(pred), 100, np.int64) if mx == 0 else 100 - (100 * c) // mx) * w
    total = 0.0 + ((0.0 + sc.astype(np.float64)) + term[pred])
    keep = cand[pred]
    pos = np.arange(len(pred))[keep]
    order = pred[keep][np.lexsort((pos, -total[keep]))]  # score descending, then scan position
    return [int(n) for n in order], mx


CHAIN = [(N, L) for N in (1, 33, 1000, 25_600, 25_601, 200_000) for L in (1, 3)]


@pytest.mark.parametrize("N,L", CHAIN)
def test_nta_soft_chain_vs_numpy(H, N, L):
    """The stored term of every candidate, then every hand-out in total_score order (TaintToleration's normalised score
    plus the term), ties by scan position; with and without sampling, on both pick kernels where N allows the
    shared-memory one."""
    R = 2
    rng = np.random.default_rng(N * 17 + L)
    member, alloc, used = _tree(N, L, R, rng)
    req, has, dw = _preemptor(R, rng)
    _edge(alloc, used, req, has, rng)
    soft = rng.integers(0, 3, N).astype(np.uint32)
    cstat = (rng.random(N) < 0.8).astype(np.uint32) | (soft << np.uint32(8))
    a, keep, cand = _rank_inputs(N, R, rng, req, has, cstat)
    term = _terms(member, _hn_scores(req, has, dw, alloc, used), TIER_W[:L], 10)
    for samp_args in (None, (50, 1, 5, N // 2 + 1)):
        for big in ((0, 1) if N <= 25_600 else (1,)):
            if N > 30_000 and samp_args is not None:
                continue  # one drain of k_evict_pick_big at this size
            term_out = np.full(N, -7.0)
            x, keep2 = _nta_args(member, alloc, used, TIER_W[:L], dw, 10, term_out)
            order = np.full(N, -7, np.int32)
            n_order = C.c_int32(0)
            word = C.c_uint64(0)
            s = SoftArgs(w_taint=3, samp=0 if samp_args is None else 1, filtered=0, big=big, seq=5, stale=0,
                         order=order.ctypes.data, n_order=C.addressof(n_order), word=C.addressof(word))
            if samp_args is not None:
                s.pct, s.min_nodes, s.min_pct, s.start = samp_args
            assert H.eh_nta_soft_chain(C.byref(a), C.byref(s), C.byref(x)) == 0
            assert np.array_equal(term_out[cand], term[cand]) and np.all(term_out[~cand] == 0.0), (N, L, samp_args, big)
            want, mx = _chain_expected(cstat, soft, cand, term, 3, samp_args)
            assert [int(v) for v in order[:n_order.value]] == want, (N, L, samp_args, big)
            assert word.value == (5 << 8) | mx


def _apply_restated(used, member, node, victims, rt_req, rt_has, req, has, undo):
    """Statement.Evict of the victims, then Statement.Pipeline (undo: UnPipeline, then unevict in reverse order), each a
    Deallocate / Allocate event on every level's hypernode of the node"""
    used = used.copy()
    R = used.shape[0]

    def book(vec, bits, sign):
        for l in range(member.shape[0]):
            h = member[l, node]
            if h < 0:
                continue
            for d in range(R):
                if d < 2 or (bits >> d) & 1:
                    used[d, h] = used[d, h] + sign * vec[d]
    sg = -1.0 if undo else 1.0
    if undo:
        book(req, has, sg)
    for r in (victims[::-1] if undo else victims):
        book(rt_req[:, r], int(rt_has[r]), -sg)
    if not undo:
        book(req, has, sg)
    return used


@pytest.mark.parametrize("R,L,integral", [(2, 1, True), (2, 3, True), (10, 2, True), (10, 3, False), (3, 2, False)])
def test_nta_apply_and_undo(H, R, L, integral):
    """hyperNodeResourceCache.used after k_evict_apply<true> and after its undo equals the restatement bit for bit;
    with integer-valued requests the undo gives back the opening bits."""
    rng = np.random.default_rng(R * 10 + L + integral)
    N, RT = 40, 60
    member, alloc, used0 = _tree(N, L, R, rng)
    if integral:
        used0 = np.floor(used0)
    rt_req = rng.integers(1, 5, (R, RT)).astype(np.float64) if integral else rng.uniform(0.1, 4.0, (R, RT))
    rt_has = (rng.integers(0, 1 << R, RT).astype(np.uint32) | 3)
    req = rng.integers(1, 5, R).astype(np.float64) if integral else rng.uniform(0.1, 4.0, R)
    has = int(rng.integers(0, 1 << R)) | 3
    for node in (0, 17, N - 1):
        node_in = any(member[l, node] >= 0 for l in range(L))
        victims = np.array(rng.choice(RT, 5, replace=False), np.int32)
        rows = dict(rel=np.zeros((R, N)), pip=np.zeros((R, N)), kreq=np.zeros((1, N)), knz=np.zeros((2, N)),
                    pod_count=np.zeros(N, np.int32), rt_evicted=np.zeros(RT, np.uint8), rt_req=np.ascontiguousarray(rt_req),
                    rt_kreq=np.zeros((1, RT)), rt_knz=np.zeros((2, RT)), req=req, kreq_t=np.zeros(1), knz_t=np.zeros(2),
                    victims=victims)
        used = np.ascontiguousarray(used0.copy())
        x = NtaApply(L=L, H=used.shape[1], member=np.ascontiguousarray(member).ctypes.data, hn_used=used.ctypes.data,
                     rt_has=rt_has.ctypes.data, has=has)
        m = member  # keeps the array alive with x
        after = None
        for undo in (0, 1):
            a = ApplyArgs(N=N, R=R, K=1, RT=RT, has_predicates=0, node=node, n_victims=len(victims), undo=undo)
            for k, v in rows.items():
                setattr(a, k, v.ctypes.data)
            want = _apply_restated(used0 if undo == 0 else after, m, node, victims, rt_req, rt_has, req, has, undo)
            assert H.eh_apply_nta(C.byref(a), C.byref(x)) == 0
            assert np.array_equal(used.view(np.uint64), want.view(np.uint64)), (R, L, node, undo)
            if undo == 0:
                assert np.array_equal(used, used0) != node_in, (R, L, node)  # the statement moved the node's hypernodes
            after = used.copy()
        if integral:
            assert np.array_equal(used.view(np.uint64), used0.view(np.uint64)), (R, L, node)


def test_nta_entry_points_reject_bad_tables(H):
    rng = np.random.default_rng(3)
    N, R = 8, 2
    member, alloc, used = _tree(N, 1, R, rng)
    req, has, dw = _preemptor(R, rng)
    a, keep, _ = _rank_inputs(N, R, rng, req, has, np.ones(N, np.uint32))
    bad = member.copy()
    bad[0, 3] = alloc.shape[1]  # a hypernode index out of range
    x, keep2 = _nta_args(bad, alloc, used, TIER_W[:1], dw, 10, np.zeros(N))
    assert H.eh_nta_rank(C.byref(a), C.byref(x)) == -1
    x, keep3 = _nta_args(member, alloc, used, TIER_W[:1], dw, 10, np.zeros(N))
    x.L = abi.VC_MAX_TIERS + 1
    assert H.eh_nta_rank(C.byref(a), C.byref(x)) == -1
