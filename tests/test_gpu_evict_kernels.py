"""The preempt / reclaim kernels of volcano_b200/csrc/vc_evict.cuh launched on their own (tools/kernels/evict_harness.cu,
built by build()) and compared with exact references:
  k_evict_pick / k_evict_pick_big  the hand-out order against numpy.lexsort, drained launch by launch like the host loop;
  k_evict_rank                     the candidate flags against a restatement of the filter in Python with exact sums;
  k_evict_apply                    the node rows after apply and after undo against a float64 restatement of
                                   Statement.Evict / Pipeline / Discard.
The end-to-end tests only see the pick order through the first node where an eviction succeeds; these see all of it."""
import ctypes as C
import os
import random
from fractions import Fraction

import numpy as np
import pytest

from volcano_b200 import abi

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "tools", "kernels", "_build", "evict_harness.so")
EV_PICK_K, EV_MAX_VICTIMS = 32, 256
PREEMPT, INTRA, RECLAIM = 0, 1, 2
MIN_RES = 0.1  # VC_MIN_RESOURCE, api/resource_info.go:45-47
_p = C.c_void_p


class RankArgs(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("N", "R", "RT", "J", "Q", "pods_dim", "exact_sums", "n_plugins")] + \
               [(n, _p) for n in ("plugin", "tier", "enabled", "idle", "rel", "pip", "cstat", "rt_off", "rt_idx", "rt_req",
                                  "rt_flags", "rt_job", "rt_prio", "rt_evicted", "j_queue", "j_prio", "j_min", "j_ready",
                                  "q_flags", "q_over")] + \
               [(n, C.c_int) for n in ("mode", "job", "queue", "job_prio", "task_prio")] + \
               [("req", _p), ("has", C.c_uint32), ("quota_on", C.c_int), ("quota_open", C.c_int), ("qalloc_has", C.c_uint32),
                ("qdes_has", C.c_uint32), ("qalloc", _p), ("qdes", _p), ("cand", _p), ("key", _p)]


class ApplyArgs(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("N", "R", "K", "RT", "has_predicates")] + \
               [(n, _p) for n in ("rel", "pip", "kreq", "knz", "pod_count", "rt_evicted", "rt_req", "rt_kreq", "rt_knz", "req",
                                  "kreq_t", "knz_t")] + \
               [("node", C.c_int), ("n_victims", C.c_int), ("victims", _p), ("undo", C.c_int)]


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build() compiles it")
    L = C.CDLL(LIB)
    L.eh_pick_open.argtypes = [C.c_int, _p, _p, C.POINTER(_p)]
    L.eh_pick_close.argtypes = [_p]
    L.eh_pick_launch.argtypes = [_p, C.c_int, C.c_int, C.c_int, _p, _p]
    L.eh_rank.argtypes = [C.POINTER(RankArgs)]
    L.eh_apply.argtypes = [C.POINTER(ApplyArgs)]
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data


def score_key(x):
    """ev_score_key: the order-preserving map of a double onto uint64."""
    u = np.asarray(x, np.float64).view(np.uint64)
    return np.where(u >> np.uint64(63) != 0, ~u, u | np.uint64(1 << 63)).astype(np.uint64)


# ---- pick ------------------------------------------------------------------------------------------------------------
def _drain(H, cand0, key, big, mode):
    """Relaunch until a batch is short or -1-terminated, checking every launch; returns the concatenated hand-outs."""
    N = len(cand0)
    live = np.flatnonzero(cand0 == 1)
    ref = live if mode == RECLAIM else live[np.lexsort((live, ~key[live]))]  # key descending, node ascending
    h = _p()
    assert H.eh_pick_open(N, _ptr(cand0), _ptr(key), C.byref(h)) == 0
    words = np.zeros(EV_PICK_K + 1, np.int32)
    cand = np.zeros(N, np.uint8)
    got = []
    want_cand = cand0.copy()
    try:
        for seq in range(1, len(ref) // EV_PICK_K + 3):
            assert H.eh_pick_launch(h, big, mode, seq, _ptr(words), _ptr(cand)) == 0
            assert words[EV_PICK_K] == seq  # the sequence word is the launch's last store
            batch = words[:EV_PICK_K]
            n = int(np.argmax(batch < 0)) if (batch < 0).any() else EV_PICK_K
            assert (batch[n:] == -1).all(), batch
            assert batch[:n].tolist() == ref[len(got):len(got) + n].tolist(), (len(got), batch[:n], ref[len(got):len(got) + n])
            got.extend(batch[:n].tolist())
            want_cand[batch[:n]] = 2
            assert np.array_equal(cand, want_cand)
            if n < EV_PICK_K:
                break
        else:
            pytest.fail("the pick kernel never ran out of candidates")
    finally:
        H.eh_pick_close(h)
    assert len(got) == len(ref) and len(set(got)) == len(got)
    return got


KEY_SCORES = np.array([-1e300, -7.5, -1.0, -5e-324, -0.0, 0.0, 5e-324, 2.2250738585072014e-308 / 3, 1.0, 3.0, 100.0,
                       1e300, np.inf, -np.inf])


def _pick_cases(N, rng):
    """(name, cand, key) for N nodes: candidate densities from one node to every node, counts around multiples of 32,
    ties over warps and over several nodes per lane, a single warp holding every candidate, every warp holding 32."""
    def mk(sel, keys="mixed", tried=0):
        cand = np.zeros(N, np.uint8)
        cand[sel] = 1
        if tried:  # nodes tried earlier (cand 2) are never handed out again
            cand[rng.choice(N, min(tried, N), replace=False)] = 2
        if keys == "equal":
            key = np.full(N, score_key(0.0), np.uint64)
        elif keys == "few":
            key = score_key(rng.choice([-1.0, 0.0, 2.0], N))
        else:
            key = score_key(rng.choice(KEY_SCORES, N))
        return cand, key
    out = [("one", mk([rng.integers(N)])), ("last", mk([N - 1], "equal"))]
    for c in (31, 32, 33, 32 * 7 + 5):
        if c <= N:
            out.append((f"n{c}", mk(rng.choice(N, c, replace=False))))
            out.append((f"n{c}-tied", mk(rng.choice(N, c, replace=False), "equal")))
    if N <= 30_000:  # every node: hundreds of launches each
        out += [("all-equal", mk(np.arange(N), "equal")), ("all-mixed", mk(np.arange(N), "mixed", tried=N // 9)),
                ("all-few", mk(np.arange(N), "few"))]
    else:
        out += [("strided-equal", mk(np.arange(0, N, 37), "equal")), ("dense-few", mk(rng.choice(N, 20_000, replace=False), "few"))]
    if N >= 1024:
        owner_warp = (np.arange(N) % 1024) // 32
        w = int(rng.integers(32))
        out.append(("one-warp", mk(np.flatnonzero(owner_warp == w), "few")))
        out.append(("one-warp-equal", mk(np.flatnonzero(owner_warp == w), "equal")))
        per = [rng.choice(np.flatnonzero(owner_warp == x), 32, replace=False) for x in range(32)]
        out.append(("warps-32", mk(np.concatenate(per), "few")))
        out.append(("warps-32-equal", mk(np.concatenate(per), "equal")))
    return out


PICK_NS = [1, 31, 32, 33, 1023, 1024, 1025, 4097, 25_600, 25_601, 200_000]


@pytest.mark.parametrize("N", PICK_NS)
def test_pick_order_vs_lexsort(H, N):
    """Both pick kernels (k_evict_pick while the keys fit in shared memory) against the reference order, preempt and
    reclaim, every launch of the drain checked."""
    rng = np.random.default_rng(N)
    cached = N <= H.eh_pick_smem_max_nodes()
    assert cached == (N * 8 <= 200 * 1024)
    for name, (cand, key) in _pick_cases(N, rng):
        for mode in (PREEMPT, RECLAIM):
            for big in ((0, 1) if cached else (1,)):
                try:
                    _drain(H, cand, key, big, mode)
                except AssertionError as e:
                    raise AssertionError(f"N={N} case={name} mode={mode} big={big}: {e}") from None


def test_pick_rejects_out_of_range(H):
    """The cached kernel's shared-memory bound and the other arguments are checked before any launch."""
    n = H.eh_pick_smem_max_nodes() + 1
    cand, key = np.ones(n, np.uint8), np.zeros(n, np.uint64)
    h = _p()
    assert H.eh_pick_open(n, _ptr(cand), _ptr(key), C.byref(h)) == 0
    words = np.zeros(EV_PICK_K + 1, np.int32)
    try:
        assert H.eh_pick_launch(h, 0, PREEMPT, 1, _ptr(words), None) == -1
        assert H.eh_pick_launch(h, 1, 3, 1, _ptr(words), None) == -1
    finally:
        H.eh_pick_close(h)
    bad = np.array([0, 3], np.uint8)
    assert H.eh_pick_open(2, _ptr(bad), _ptr(key), C.byref(h)) == -1


# ---- rank ------------------------------------------------------------------------------------------------------------
VOTERS = [abi.VC_PLUGIN_CONFORMANCE, abi.VC_PLUGIN_GANG, abi.VC_PLUGIN_PRIORITY, abi.VC_PLUGIN_DRF, abi.VC_PLUGIN_PROPORTION]


def _rank_case(seed, N, R, tasks_per_node, integral, mode):
    rng = np.random.default_rng(seed)
    rnd = random.Random(seed)
    J, Q = 6, 4
    counts = np.array([tasks_per_node[i % len(tasks_per_node)] for i in range(N)], np.int32)
    rng.shuffle(counts)
    RT = int(counts.sum())
    rt_off = np.zeros(N + 1, np.int32)
    rt_off[1:] = np.cumsum(counts)
    rt_idx = rng.permutation(RT).astype(np.int32)  # node.Tasks entries need not be contiguous task ids
    if integral:
        rt_req = rng.integers(0, 3, (R, RT)).astype(np.float64)
        idle = rng.integers(0, 8, (R, N)).astype(np.float64)
        rel = rng.integers(0, 3, (R, N)).astype(np.float64)
        pip = rng.integers(0, 3, (R, N)).astype(np.float64)
        req = rng.integers(1, 6, R).astype(np.float64)
    else:
        rt_req = np.round(rng.random((R, RT)) * 3, 3) + rng.random((R, RT)) * 1e-7
        idle = rng.random((R, N)) * 4
        rel = rng.random((R, N)) * 2
        pip = np.zeros((R, N))
        req = 1.3 + rng.random(R) * 5
    has = 3 | int(sum(1 << d for d in range(2, R) if rng.random() < 3.0 / R))  # some scalar dims not requested
    rt_flags = np.zeros(RT, np.uint32)
    rt_flags |= np.where(rng.random(RT) < 0.8, abi.VC_RT_PREEMPTABLE, 0).astype(np.uint32)
    rt_flags |= np.where(rng.random(RT) < 0.8, abi.VC_RT_RUNNING, abi.VC_RT_BOUND).astype(np.uint32)
    rt_flags |= np.where(rng.random(RT) < 0.1, abi.VC_RT_CRITICAL, 0).astype(np.uint32)
    a = dict(N=N, R=R, RT=RT, J=J, Q=Q, pods_dim=(R - 1 if rng.random() < 0.5 else -1),
             idle=idle, rel=rel, pip=pip, cstat=(rng.random(N) < 0.9).astype(np.uint32),
             rt_off=rt_off, rt_idx=rt_idx, rt_req=rt_req, rt_flags=rt_flags,
             rt_job=rng.integers(-1, J, RT).astype(np.int32), rt_prio=rng.integers(0, 4, RT).astype(np.int32),
             rt_evicted=(rng.random(RT) < 0.05).astype(np.uint8), j_queue=rng.integers(-1, Q, J).astype(np.int32),
             j_prio=rng.integers(0, 4, J).astype(np.int32), j_min=rng.integers(0, 4, J).astype(np.int32),
             j_ready=rng.integers(0, 6, J).astype(np.int32),
             q_flags=np.where(rng.random(Q) < 0.3, abi.VC_QUEUE_NOT_RECLAIMABLE, 0).astype(np.uint32),
             q_over=(rng.random(Q) < 0.6).astype(np.uint8), mode=mode, job=int(rng.integers(0, J)),
             job_prio=int(rng.integers(0, 4)), task_prio=int(rng.integers(0, 4)), req=req, has=has)
    a["queue"] = int(a["j_queue"][a["job"]]) if a["j_queue"][a["job"]] >= 0 else 0
    # tiers of voters, random subsets and splits; sometimes a tier whose last voter says no to most tasks
    pl = [v for v in VOTERS if rnd.random() < 0.8] or [abi.VC_PLUGIN_GANG]
    rnd.shuffle(pl)
    if rnd.random() < 0.3:  # priority last in the first tier: a "no" for every task of equal or higher priority
        pl = [p for p in pl if p != abi.VC_PLUGIN_PRIORITY] + [abi.VC_PLUGIN_PRIORITY]
        split = len(pl)
    else:
        split = rnd.randint(0, len(pl))
    tiers = [0 if i < split else 1 for i in range(len(pl))]
    en = [rnd.choice([abi.VC_EN_PREEMPTABLE | abi.VC_EN_RECLAIMABLE, abi.VC_EN_PREEMPTABLE, abi.VC_EN_RECLAIMABLE, 0])
          for _ in pl]
    a.update(plugin=np.array(pl, np.int32), tier=np.array(tiers, np.int32), enabled=np.array(en, np.uint32))
    quota_on = integral and mode != RECLAIM and rnd.random() < 0.5
    a.update(quota_on=int(quota_on), quota_open=int(rnd.random() < 0.8), qalloc_has=int(rng.integers(0, 1 << R)),
             qdes_has=int(rng.integers(0, 1 << R)), qalloc=rng.integers(0, 30, R).astype(np.float64),
             qdes=rng.integers(5, 40, R).astype(np.float64))
    a["exact_sums"] = int(integral)
    return a


def _filter(a, r):
    """ev_filter: may the action consider running task r at all (preempt.go:198-214, :252-268, reclaim.go:184-199)?"""
    if a["rt_evicted"][r]:
        return False
    f = int(a["rt_flags"][r])
    if not f & abi.VC_RT_PREEMPTABLE:
        return False
    j = int(a["rt_job"][r])
    if a["mode"] == RECLAIM:
        if not f & abi.VC_RT_RUNNING or j < 0:
            return False
        q = int(a["j_queue"][j])
        return q >= 0 and q != a["queue"] and not a["q_flags"][q] & abi.VC_QUEUE_NOT_RECLAIMABLE
    if not f & (abi.VC_RT_RUNNING | abi.VC_RT_BOUND):
        return False
    if a["mode"] == INTRA:
        return j == a["job"]
    return j >= 0 and j != a["job"] and a["j_queue"][j] == a["queue"]


def _may_be_victim(a, r):
    """Only the last voting plugin of the deciding tier is certain about a victim (session_plugins.go:211-307)."""
    reclaim = a["mode"] == RECLAIM
    flag = abi.VC_EN_RECLAIMABLE if reclaim else abi.VC_EN_PREEMPTABLE
    j = int(a["rt_job"][r])
    tiers = {}
    for pl, tier, en in zip(a["plugin"], a["tier"], a["enabled"]):
        if not en & flag:
            continue
        if pl == abi.VC_PLUGIN_CONFORMANCE:
            vote = not a["rt_flags"][r] & abi.VC_RT_CRITICAL
        elif pl == abi.VC_PLUGIN_GANG:
            vote = j >= 0 and a["j_ready"][j] > a["j_min"][j]
        elif pl == abi.VC_PLUGIN_PRIORITY and not reclaim:
            vote = j >= 0 and (a["j_prio"][j] < a["job_prio"] if j != a["job"] else a["rt_prio"][r] < a["task_prio"])
        elif pl == abi.VC_PLUGIN_DRF and not reclaim:
            vote = j >= 0
        elif pl == abi.VC_PLUGIN_PROPORTION and reclaim:
            vote = j >= 0 and a["j_queue"][j] >= 0 and bool(a["q_over"][a["j_queue"][j]])
        else:
            continue
        tiers[int(tier)] = bool(vote)  # the tier's last voter so far
    return any(tiers.values())


def _le_eps(l, r):
    return l < r or abs(l - r) < Fraction(MIN_RES)


def _rank_ref(a, slack=0.0):
    """(cand, have) per node with exact sums: cand as the kernel must flag it when the sums are exact; with `slack` the
    relative tolerance the kernel grants inexact sums."""
    N, R = a["N"], a["R"]
    cand = np.zeros(N, np.uint8)
    for n in range(N):
        if not a["cstat"][n] & 1:
            continue
        n_pass = 0
        freed = [Fraction(0)] * R
        for k in range(a["rt_off"][n], a["rt_off"][n + 1]):
            r = int(a["rt_idx"][k])
            if not _filter(a, r):
                continue
            n_pass += 1
            if _may_be_victim(a, r):
                for d in range(R):
                    freed[d] += Fraction(float(a["rt_req"][d, r]))
        fits = True
        for d in range(R):
            if d >= 2 and not a["has"] >> d & 1:
                continue
            pot = (a["idle"][d, n] + a["rel"][d, n]) - a["pip"][d, n]  # FutureIdle, as the kernel forms it
            have = Fraction(float(pot)) + freed[d]
            if not _le_eps(Fraction(float(a["req"][d])), have + abs(have) * Fraction(slack)):
                fits = False
        if a["quota_on"] and a["exact_sums"] and a["mode"] != RECLAIM:
            if not a["quota_open"]:
                fits = False
            for d in range(R):
                rq = float(a["req"][d])
                if not rq > 0.0 or (d >= 2 and (not (a["has"] & ~3) >> d & 1 or d == a["pods_dim"])):
                    continue
                al = a["qalloc"][d] if d < 2 or a["qalloc_has"] >> d & 1 else 0.0
                de = a["qdes"][d] if d < 2 or a["qdes_has"] >> d & 1 else 0.0
                if (Fraction(float(al)) - freed[d]) + Fraction(rq) > Fraction(float(de)):
                    fits = False
        if fits and (a["mode"] != RECLAIM or n_pass > 0):
            cand[n] = 1
    return cand


def _run_rank(H, a):
    N = a["N"]
    cand, key = np.full(N, 77, np.uint8), np.full(N, 7, np.uint64)
    keep = {k: np.ascontiguousarray(v) for k, v in a.items() if isinstance(v, np.ndarray)}
    s = RankArgs()
    for name, _ in RankArgs._fields_:
        if name in keep:
            setattr(s, name, _ptr(keep[name]))
        elif name == "n_plugins":
            s.n_plugins = len(a["plugin"])
        elif name in ("cand", "key"):
            pass
        else:
            setattr(s, name, int(a[name]))
    s.cand, s.key = _ptr(cand), _ptr(key)
    return H.eh_rank(C.byref(s)), cand, key


RANK_SHAPES = [(37, 2, (0, 1, 15, 16, 17)), (101, 3, (16, 17, 33)), (53, 8, (0, 15, 33, 300)), (29, 9, (1, 16, 17, 300)),
               (45, 16, (0, 1, 15, 16, 17, 33))]


@pytest.mark.parametrize("N,R,tpn", RANK_SHAPES)
@pytest.mark.parametrize("mode", [PREEMPT, INTRA, RECLAIM])
def test_rank_flags_integral_vs_exact(H, N, R, tpn, mode):
    """Integer-valued requests (exact_sums): the candidate flags equal the exact restatement; every candidate's key is
    ev_score_key(+0.0) in preempt and 0 in reclaim (no node-order plugin); non-candidates carry key 0."""
    n_cand = 0
    for seed in range(6):
        a = _rank_case(1000 * R + 10 * mode + seed, N, R, tpn, True, mode)
        rc, cand, key = _run_rank(H, a)
        assert rc == 0
        want = _rank_ref(a)
        assert np.array_equal(cand, want), (seed, np.flatnonzero(cand != want))
        k1 = np.uint64(score_key(0.0)) if mode != RECLAIM else np.uint64(0)
        assert np.array_equal(key, np.where(want == 1, k1, np.uint64(0)).astype(np.uint64))
        n_cand += int(want.sum())
    assert 0 < n_cand < 6 * N  # both outcomes occur


@pytest.mark.parametrize("N,R,tpn", RANK_SHAPES)
def test_rank_flags_nonintegral_superset(H, N, R, tpn):
    """Non-integer requests: the kernel's filter must stay a necessary condition, so its candidates include every node
    the exact test passes, and any extra node is within the 1e-9 relative slack. Half the nodes are placed on the
    boundary (exact FutureIdle + freed just above request - 0.1), where a rounded-down sum would drop them."""
    for seed, mode in ((1, PREEMPT), (2, RECLAIM), (3, INTRA)):
        a = _rank_case(7000 * R + seed, N, R, tpn, False, mode)
        exact = _rank_ref(a)
        for n in range(0, N, 2):  # boundary nodes: idle so that have - (req - 0.1) is one ulp-ish above zero
            freed = [Fraction(0)] * R
            for k in range(a["rt_off"][n], a["rt_off"][n + 1]):
                r = int(a["rt_idx"][k])
                if _filter(a, r) and _may_be_victim(a, r):
                    for d in range(R):
                        freed[d] += Fraction(float(a["rt_req"][d, r]))
            for d in range(R):
                a["rel"][d, n] = a["pip"][d, n] = 0.0
                target = Fraction(float(a["req"][d])) - Fraction(MIN_RES) - freed[d]
                a["idle"][d, n] = np.nextafter(float(target), np.inf) if Fraction(float(target)) <= target else float(target)
        exact = _rank_ref(a)
        loose = _rank_ref(a, slack=2e-9)
        rc, cand, _ = _run_rank(H, a)
        assert rc == 0
        assert not (exact.astype(bool) & (cand != 1)).any(), ("dropped", seed, np.flatnonzero(exact.astype(bool) & (cand != 1)))
        assert not ((cand == 1) & ~loose.astype(bool)).any(), ("beyond slack", seed)
        assert exact[::2].sum() > 0


def test_rank_rejects_out_of_range(H):
    a = _rank_case(5, 20, 3, (2,), True, PREEMPT)
    a["rt_idx"] = a["rt_idx"].copy()
    a["rt_idx"][0] = a["RT"]
    assert _run_rank(H, a)[0] == -1
    a = _rank_case(5, 20, 3, (2,), True, PREEMPT)
    a["R"] = 17  # above VC_MAX_DIMS
    assert _run_rank(H, a)[0] == -1
    a = _rank_case(5, 20, 3, (2,), True, PREEMPT)
    a["enabled"] = a["enabled"] | np.uint32(abi.VC_EN_NODE_ORDER)  # no scoring rows in the harness
    assert _run_rank(H, a)[0] == -1


# ---- apply -----------------------------------------------------------------------------------------------------------
def _apply_case(rng, N, R, K, RT, integral):
    f = (lambda *s: rng.integers(0, 50, s).astype(np.float64)) if integral else (lambda *s: rng.random(s) * 50)
    return dict(rel=f(R, N), pip=f(R, N), kreq=f(K, N), knz=f(2, N), pod_count=rng.integers(300, 400, N).astype(np.int32),
                rt_evicted=np.zeros(RT, np.uint8), rt_req=f(R, RT), rt_kreq=f(K, RT), rt_knz=f(2, RT), req=f(R), kreq_t=f(K),
                knz_t=f(2))


def _run_apply(H, c, node, victims, undo, has_predicates=1):
    out = {k: c[k].copy() for k in ("rel", "pip", "kreq", "knz", "pod_count", "rt_evicted")}
    R, N = c["rel"].shape
    s = ApplyArgs(N=N, R=R, K=c["kreq"].shape[0], RT=len(c["rt_evicted"]), has_predicates=has_predicates, node=node,
                  n_victims=len(victims), undo=undo)
    vic = np.ascontiguousarray(victims, np.int32)
    for k in ("rel", "pip", "kreq", "knz", "pod_count", "rt_evicted"):
        setattr(s, k, _ptr(out[k]))
    for k in ("rt_req", "rt_kreq", "rt_knz", "req", "kreq_t", "knz_t"):
        setattr(s, k, _ptr(c[k]))
    s.victims = _ptr(vic)
    rc = H.eh_apply(C.byref(s))
    return rc, out


def _apply_ref(c, node, victims, undo):
    """Statement.Evict per victim (Releasing += Resreq; predicates RemovePod), then Statement.Pipeline; undo is
    Statement.Discard: UnPipeline, then unevict in reverse order (framework/statement.go:357-381)."""
    o = {k: c[k].copy() for k in ("rel", "pip", "kreq", "knz", "pod_count", "rt_evicted")}
    n = node

    def evict(r, s):
        o["rel"][:, n] += s * c["rt_req"][:, r]
        o["kreq"][:, n] -= s * c["rt_kreq"][:, r]
        o["knz"][:, n] -= s * c["rt_knz"][:, r]
        o["pod_count"][n] -= s
        o["rt_evicted"][r] = 1 if s > 0 else 0

    def pipeline(s):
        o["pip"][:, n] += s * c["req"]
        o["kreq"][:, n] += s * c["kreq_t"]
        o["knz"][:, n] += s * c["knz_t"]
        o["pod_count"][n] += s
    if not undo:
        for r in victims:
            evict(r, 1)
        pipeline(1)
    else:
        pipeline(-1)
        for r in reversed(victims):
            evict(r, -1)
    return o


@pytest.mark.parametrize("nv", [1, 2, 255, 256])
@pytest.mark.parametrize("integral", [True, False])
def test_apply_and_undo_vs_statement(H, nv, integral):
    rng = np.random.default_rng(nv + 1000 * integral)
    N, R, K, RT = 5, 9, 3, 300
    c = _apply_case(rng, N, R, K, RT, integral)
    node = 3
    victims = rng.choice(RT, nv, replace=False).astype(np.int32).tolist()
    rc, after = _run_apply(H, c, node, victims, 0)
    assert rc == 0
    want = _apply_ref(c, node, victims, 0)
    for k in want:
        assert np.array_equal(after[k], want[k]), k
    c2 = dict(c, **after)
    rc, back = _run_apply(H, c2, node, victims, 1)
    assert rc == 0
    want_back = _apply_ref(c2, node, victims, 1)  # the oracle's estmt_discard order
    for k in want_back:
        assert np.array_equal(back[k], want_back[k]), k
    if integral:  # apply + undo restores every row bit for bit
        for k in want_back:
            assert np.array_equal(back[k], c[k]), k
    assert (back["rt_evicted"] == 0).all()
    # without the predicates plugin the k8s rows and the pod count stay
    rc, plain = _run_apply(H, c, node, victims, 0, has_predicates=0)
    assert rc == 0
    for k in ("kreq", "knz", "pod_count"):
        assert np.array_equal(plain[k], c[k]), k
    assert np.array_equal(plain["rel"], want["rel"]) and np.array_equal(plain["pip"], want["pip"])


def test_apply_rejects_out_of_range(H):
    rng = np.random.default_rng(3)
    c = _apply_case(rng, 4, 3, 2, 300, True)
    assert _run_apply(H, c, 0, list(range(257)), 0)[0] == -1  # EV_MAX_VICTIMS
    assert _run_apply(H, c, 4, [0], 0)[0] == -1
    assert _run_apply(H, c, 0, [300], 0)[0] == -1
