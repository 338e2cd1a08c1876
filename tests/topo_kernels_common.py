"""Random dry-run instances of topology-aware preemption, their ctypes form (tools/kernels/topo_args.h), and an exact
Python restatement of SelectVictimsOnNode (actions/preempt/preempt.go:708-842) and of the candidate pick (:581-607,
:846-979) to compare the kernels and the CPU shim with. Python floats are IEEE doubles and the restatement performs the
reference's operations in its order, so results must be equal bit for bit."""
from __future__ import annotations

import ctypes as C

import numpy as np

from volcano_b200 import abi

_p = C.POINTER
VOTERS = [abi.PLUGIN_IDS[n] for n in ("gang", "conformance", "priority", "drf")]
START_UNSET = abi.VC_START_TIME_UNSET


class EhTopoArgs(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("N", "R", "J", "RT", "pods_dim", "n_plugins", "task_order_prio")] + [
        ("plugin", _p(C.c_int32)), ("tier", _p(C.c_int32)), ("enabled", _p(C.c_uint32)),
        ("idle", _p(C.c_double)), ("rel", _p(C.c_double)), ("pip", _p(C.c_double)), ("pred", _p(C.c_uint8)),
        ("rt_off", _p(C.c_int32)), ("rt_idx", _p(C.c_int32)), ("rt_req", _p(C.c_double)),
        ("rt_has", _p(C.c_uint32)), ("rt_flags", _p(C.c_uint32)), ("rt_uid", _p(C.c_uint32)),
        ("rt_job", _p(C.c_int32)), ("rt_prio", _p(C.c_int32)), ("rt_pod_prio", _p(C.c_int32)),
        ("rt_podidx", _p(C.c_int64)), ("rt_ts", _p(C.c_int64)), ("rt_start", _p(C.c_int64)), ("rt_evicted", _p(C.c_uint8)),
        ("j_queue", _p(C.c_int32)), ("j_prio", _p(C.c_int32)), ("j_min", _p(C.c_int32)), ("j_ready", _p(C.c_int32)),
        ("j_pbe", _p(C.c_int32)), ("j_rank", _p(C.c_uint32)), ("j_alloc", _p(C.c_double)), ("j_share", _p(C.c_double)),
        ("total", _p(C.c_double)), ("total_has", C.c_uint32),
        ("job", C.c_int32), ("queue", C.c_int32), ("intra", C.c_int32), ("job_prio", C.c_int32), ("task_prio", C.c_int32),
        ("req", _p(C.c_double)), ("has", C.c_uint32),
        ("sim_update", C.c_int32), ("sim_state", C.c_int32), ("sim_alloc", C.c_int32), ("q_exists", C.c_int32),
        ("qalloc", _p(C.c_double)), ("qdes", _p(C.c_double)), ("qalloc_has", C.c_uint32), ("qdes_has", C.c_uint32),
        ("qalloc_nil", C.c_int32), ("now_ns", C.c_int64),
        ("ok", _p(C.c_uint8)), ("nv", _p(C.c_int32)), ("key", _p(C.c_longlong)), ("victims", _p(C.c_int32))]


class EhSelectArgs(C.Structure):
    _fields_ = [("N", C.c_int32), ("RT", C.c_int32), ("pred", _p(C.c_uint8)), ("ok", _p(C.c_uint8)),
                ("nv", _p(C.c_int32)), ("key", _p(C.c_longlong)), ("rt_off", _p(C.c_int32)), ("victims", _p(C.c_int32)),
                ("seed_k", C.c_uint64), ("pct", C.c_int32), ("min_abs", C.c_int32), ("max_abs", C.c_int32),
                ("seq", C.c_int32), ("words", _p(C.c_int32))]


def random_instance(rng, N, R, max_pods=300, heavy=2, non_integer=False):
    """N nodes, most running 0-8 pods, `heavy` of them up to max_pods; R resource dimensions; random voter tiers."""
    I = {"N": N, "R": R}
    pods = rng.integers(0, 9, N)
    if N and heavy:
        pods[rng.choice(N, min(heavy, N), replace=False)] = rng.integers(max_pods // 2, max_pods + 1, min(heavy, N))
    off = np.zeros(N + 1, np.int32)
    off[1:] = np.cumsum(pods)
    RT = int(off[-1])
    J = int(rng.integers(2, 9))
    I.update(RT=RT, J=J, rt_off=off, rt_idx=rng.permutation(RT).astype(np.int32))
    I["pods_dim"] = int(rng.integers(2, R)) if R > 2 and rng.random() < 0.5 else -1

    def amounts(shape, hi):
        a = rng.integers(0, hi, shape).astype(np.float64)
        return a + (rng.integers(0, 10, shape) * 0.1 if non_integer else 0.0)
    I["rt_req"] = amounts((R, RT), 4)
    I["rt_has"] = (rng.integers(0, 1 << R, RT, dtype=np.int64) & ~3).astype(np.uint32)
    fl = np.where(rng.random(RT) < 0.85, abi.VC_RT_PREEMPTABLE, 0)
    fl |= np.where(rng.random(RT) < 0.8, abi.VC_RT_RUNNING, abi.VC_RT_BOUND)
    fl |= np.where(rng.random(RT) < 0.1, abi.VC_RT_CRITICAL, 0)
    I["rt_flags"] = fl.astype(np.uint32)
    I["rt_uid"] = rng.permutation(RT).astype(np.uint32)
    I["rt_job"] = rng.integers(-1, J, RT).astype(np.int32) if rng.random() < 0.3 else rng.integers(0, J, RT).astype(np.int32)
    I["rt_prio"] = rng.integers(0, 4, RT).astype(np.int32)
    I["rt_pod_prio"] = rng.choice([-5, 0, 3, 10, 100000], RT).astype(np.int32)
    I["rt_podidx"] = np.where(rng.random(RT) < 0.5, -1, rng.integers(0, 6, RT)).astype(np.int64)  # indexed and not mixed
    I["rt_ts"] = rng.integers(0, 4, RT).astype(np.int64)
    I["rt_start"] = np.where(rng.random(RT) < 0.2, START_UNSET, rng.integers(0, 4, RT) * 10 ** 9).astype(np.int64)
    I["rt_evicted"] = (rng.random(RT) < 0.05).astype(np.uint8)
    I["idle"] = amounts((R, N), 3)
    I["rel"] = np.where(rng.random((R, N)) < 0.2, amounts((R, N), 2), 0.0)
    I["pip"] = np.where(rng.random((R, N)) < 0.2, amounts((R, N), 2), 0.0)
    I["pred"] = (rng.random(N) < 0.9).astype(np.uint8)
    I["j_queue"] = rng.integers(0, 2, J).astype(np.int32)
    I["j_prio"] = rng.choice([0, 10, 100], J).astype(np.int32)
    I["j_min"] = rng.integers(0, 4, J).astype(np.int32)
    I["j_ready"] = rng.integers(0, 8, J).astype(np.int32)
    I["j_pbe"] = rng.integers(0, 2, J).astype(np.int32)
    I["j_rank"] = rng.permutation(J).astype(np.uint32)
    I["j_alloc"] = amounts((R, J), 30)
    I["j_share"] = rng.choice([0.0, 0.25, 0.5], J)
    I["total"] = amounts(R, 200) + 1.0
    I["total_has"] = int(rng.integers(0, 1 << R)) & ~3
    # tiers of voters, job-order and task-order enables
    names = [p for p in VOTERS if rng.random() < 0.7] or [VOTERS[0]]
    rng.shuffle(names)
    split = int(rng.integers(0, len(names) + 1))
    I["plugin"] = np.array(names, np.int32)
    I["tier"] = np.array([0 if i < split else 1 for i in range(len(names))], np.int32)
    en = []
    for p in names:
        e = abi.VC_EN_PREEMPTABLE if rng.random() < 0.9 else 0
        if p != abi.PLUGIN_IDS["conformance"] and rng.random() < 0.6:
            e |= abi.VC_EN_JOB_ORDER
        en.append(e)
    I["enabled"] = np.array(en, np.uint32)
    I["n_plugins"] = len(names)
    I["task_order_prio"] = int(rng.random() < 0.6)
    # the preemptor
    I["job"] = 0
    I["queue"] = int(I["j_queue"][0])
    I["intra"] = int(rng.random() < 0.3)
    I["job_prio"], I["task_prio"] = int(rng.choice([50, 1000])), int(rng.integers(0, 5))
    I["req"] = amounts(R, 4)
    I["has"] = int(sum(1 << d for d in range(2, R) if rng.random() < 0.25))
    I["sim_alloc"] = int(rng.random() < 0.6)
    I["sim_update"] = int(I["sim_alloc"] or rng.random() < 0.5)
    I["sim_state"] = int(rng.random() < 0.85)
    I["q_exists"] = int(rng.random() < 0.95)
    I["qalloc"], I["qdes"] = amounts(R, 40), amounts(R, 60)
    I["qalloc_has"], I["qdes_has"] = int(rng.integers(0, 1 << R)) & ~3, int(rng.integers(0, 1 << R)) & ~3
    I["qalloc_nil"] = int(I["qalloc_has"] == 0)
    I["now_ns"] = int(rng.integers(0, 5)) * 10 ** 9
    return I



def to_args(I):
    """-> (EhTopoArgs, outputs dict); the arrays stay referenced by the outputs dict."""
    a = EhTopoArgs()
    keep = {}
    for name, ctype in EhTopoArgs._fields_:
        if name in ("ok", "nv", "key", "victims"):
            continue
        v = I[name]
        if isinstance(v, np.ndarray):
            arr = np.ascontiguousarray(v)
            keep[name] = arr
            setattr(a, name, arr.ctypes.data_as(ctype))
        else:
            setattr(a, name, int(v))
    out = {"ok": np.zeros(max(I["N"], 1), np.uint8), "nv": np.zeros(max(I["N"], 1), np.int32),
           "key": np.zeros(4 * max(I["N"], 1), np.int64), "victims": np.zeros(max(I["RT"], 1), np.int32)}
    a.ok = out["ok"].ctypes.data_as(_p(C.c_uint8)); a.nv = out["nv"].ctypes.data_as(_p(C.c_int32))
    a.key = out["key"].ctypes.data_as(_p(C.c_longlong)); a.victims = out["victims"].ctypes.data_as(_p(C.c_int32))
    out["_keep"] = keep
    return a, out


# ---- the exact restatement ----------------------------------------------------------------------------------------
def _le(l, r):
    return l < r or abs(l - r) < 0.1


def _share(I, a):
    res = 0.0
    for d in range(I["R"]):
        if d >= 2 and not (I["total_has"] >> d) & 1:
            continue
        t = float(I["total"][d])
        if not t >= 0.1:
            continue
        sh = (0.0 if a[d] == 0 else 1.0) if t == 0 else a[d] / t
        if sh > res:
            res = sh
    return res


def _res_add(v, has, nil, rq, rq_has, R):
    v[0] += rq[0]; v[1] += rq[1]
    for d in range(2, R):
        if (rq_has >> d) & 1:
            nil = False; has |= 1 << d; v[d] += rq[d]
    return has, nil


def _res_sub(v, has, nil, rq, rq_has, R):
    v[0] -= rq[0]; v[1] -= rq[1]
    if nil:
        return has, nil
    for d in range(2, R):
        if (rq_has >> d) & 1:
            has |= 1 << d; v[d] -= rq[d]
    return has, nil


def dry_run(I, n):
    """SelectVictimsOnNode on node n -> None, or (victims in list order, the four pick scores)."""
    R, J = I["R"], I["J"]
    job, flags, req = I["rt_job"], I["rt_flags"], I["rt_req"]
    if not I["pred"][n]:
        return None

    def keep(r):
        if I["rt_evicted"][r] or not flags[r] & abi.VC_RT_PREEMPTABLE or not flags[r] & (abi.VC_RT_RUNNING | abi.VC_RT_BOUND):
            return False
        j = int(job[r])
        if I["intra"]:
            return j == I["job"]
        return j >= 0 and j != I["job"] and I["j_queue"][j] == I["queue"]
    cands = [int(I["rt_idx"][x]) for x in range(I["rt_off"][n], I["rt_off"][n + 1]) if keep(int(I["rt_idx"][x]))]

    def vote(pl):
        out = []
        if pl == abi.PLUGIN_IDS["gang"]:
            occ = {}
            for r in cands:
                j = int(job[r])
                if j < 0:
                    continue
                occ.setdefault(j, int(I["j_ready"][j]))
                if occ[j] > I["j_min"][j]:
                    occ[j] -= 1
                    out.append(r)
        elif pl == abi.PLUGIN_IDS["conformance"]:
            out = [r for r in cands if not flags[r] & abi.VC_RT_CRITICAL]
        elif pl == abi.PLUGIN_IDS["priority"]:
            for r in cands:
                j = int(job[r])
                if j < 0:
                    continue
                if (I["j_prio"][j] < I["job_prio"]) if j != I["job"] else (I["rt_prio"][r] < I["task_prio"]):
                    out.append(r)
        else:
            ls = _share(I, [float(I["j_alloc"][d, I["job"]]) + float(I["req"][d]) for d in range(R)])
            allocs = {}
            for r in cands:
                j = int(job[r])
                if j < 0:
                    continue
                ra = allocs.setdefault(j, [float(I["j_alloc"][d, j]) for d in range(R)])
                for d in range(R):
                    ra[d] -= float(req[d, r])
                rs = _share(I, ra)
                if ls < rs or abs(ls - rs) <= 0.000001:
                    out.append(r)
        return out
    victims, nil = [], True
    i, P = 0, len(I["plugin"])
    while i < P:
        tier = I["tier"][i]
        x = i
        while x < P and I["tier"][x] == tier:
            if I["enabled"][x] & abi.VC_EN_PREEMPTABLE:
                c = vote(int(I["plugin"][x]))
                if not c:
                    victims, nil = [], True
                    break
                if nil:
                    victims, nil = c, False
                else:
                    victims = [v for v in victims if v in c]
                    nil = not victims
            x += 1
        while i < P and I["tier"][i] == tier:
            i += 1
        if not nil:
            break
    for d in range(R):  # ValidateVictims
        fi = (float(I["idle"][d, n]) + float(I["rel"][d, n])) - float(I["pip"][d, n])
        for v in victims:
            fi += float(req[d, v])
        if d >= 2 and not (I["has"] >> d) & 1:
            continue
        if not _le(float(I["req"][d]), fi):
            return None

    def run_less(l, r):
        if I["task_order_prio"] and I["rt_prio"][l] != I["rt_prio"][r]:
            return I["rt_prio"][l] > I["rt_prio"][r]
        il, ir = I["rt_podidx"][l], I["rt_podidx"][r]
        if il < 0 or ir < 0 or il == ir:
            if I["rt_ts"][l] == I["rt_ts"][r]:
                return I["rt_uid"][l] < I["rt_uid"][r]
            return I["rt_ts"][l] < I["rt_ts"][r]
        return not il > ir

    def job_less(l, r):
        for p, e in zip(I["plugin"], I["enabled"]):
            if not e & abi.VC_EN_JOB_ORDER:
                continue
            c = 0
            if p == abi.PLUGIN_IDS["priority"]:
                c = -1 if I["j_prio"][l] > I["j_prio"][r] else (1 if I["j_prio"][l] < I["j_prio"][r] else 0)
            elif p == abi.PLUGIN_IDS["gang"]:
                lr = I["j_ready"][l] + I["j_pbe"][l] >= I["j_min"][l]
                rr = I["j_ready"][r] + I["j_pbe"][r] >= I["j_min"][r]
                c = 0 if (lr and rr) else (1 if lr else (-1 if rr else 0))
            elif p == abi.PLUGIN_IDS["drf"]:
                sl, sr = I["j_share"][l], I["j_share"][r]
                c = 0 if sl == sr else (-1 if sl < sr else 1)
            if c:
                return c < 0
        return I["j_rank"][l] < I["j_rank"][r]

    def less(l, r):
        return (not run_less(l, r)) if job[l] == job[r] else (not job_less(int(job[l]), int(job[r])))
    h = []  # container/heap

    def push(x):
        h.append(x)
        j = len(h) - 1
        while j > 0:
            i2 = (j - 1) // 2
            if not less(h[j], h[i2]):
                break
            h[i2], h[j] = h[j], h[i2]
            j = i2

    def pop():
        n1 = len(h) - 1
        h[0], h[n1] = h[n1], h[0]
        i2 = 0
        while True:
            j1 = 2 * i2 + 1
            if j1 >= n1:
                break
            j = j1
            if j1 + 1 < n1 and less(h[j1 + 1], h[j1]):
                j = j1 + 1
            if not less(h[j], h[i2]):
                break
            h[i2], h[j] = h[j], h[i2]
            i2 = j
        return h.pop()
    for v in victims:
        push(v)
    idle = [float(I["idle"][d, n]) for d in range(R)]
    qa = [float(x) for x in I["qalloc"]]
    qstate = [I["qalloc_has"], bool(I["qalloc_nil"])]

    def fits():
        if I["sim_alloc"]:
            if not I["sim_state"] or not I["q_exists"]:
                return False
            fu = list(qa)
            fh, fnil = _res_add(fu, qstate[0], qstate[1], [float(x) for x in I["req"]], I["has"], R)
            rq = I["req"]
            if rq[0] > 0 and fu[0] > I["qdes"][0]:
                return False
            if rq[1] > 0 and fu[1] > I["qdes"][1]:
                return False
            if not fnil:
                for d in range(2, R):
                    if not (I["has"] >> d) & 1 or d == I["pods_dim"]:
                        continue
                    lq = fu[d] if (fh >> d) & 1 else 0.0
                    rv = float(I["qdes"][d]) if (I["qdes_has"] >> d) & 1 else 0.0
                    if rq[d] > 0 and lq > rv:
                        return False
        for d in range(R):
            if d >= 2 and not (I["has"] >> d) & 1:
                continue
            if not _le(float(I["req"][d]), (idle[d] + float(I["rel"][d, n])) - float(I["pip"][d, n])):
                return False
        return True

    def remove(r):
        if I["sim_update"]:
            if not I["sim_state"] or not I["q_exists"]:
                return False
            qstate[0], qstate[1] = _res_sub(qa, qstate[0], qstate[1], [float(req[d, r]) for d in range(R)], int(I["rt_has"][r]), R)
        for d in range(R):
            idle[d] += float(req[d, r])
        return True
    popped = []
    while h:
        r = pop()
        popped.append(r)
        if not remove(r):
            return None
        if fits():
            break
    if not popped:
        return None
    out = []
    for r in reversed(popped):
        if I["sim_update"]:
            qstate[0], qstate[1] = _res_add(qa, qstate[0], qstate[1], [float(req[d, r]) for d in range(R)], int(I["rt_has"][r]), R)
        for d in range(R):
            idle[d] -= float(req[d, r])
        if not fits():
            remove(r)
            out.append(r)
    if not out:
        return None
    pp = [int(I["rt_pod_prio"][r]) for r in out]
    start = [int(I["now_ns"]) if I["rt_start"][r] == START_UNSET else int(I["rt_start"][r]) for r in out]
    earliest, maxp = start[0], pp[0]
    for p, s in zip(pp, start):
        if p == maxp:
            earliest = min(earliest, s)
        elif p > maxp:
            maxp, earliest = p, s
    return out, (-pp[0], -sum(p + 2 ** 31 for p in pp), -len(out), earliest)


def check_dry_run(I, out, nodes):
    """The launcher's outputs against the restatement on `nodes`; -> number of candidates among them."""
    N, hits = I["N"], 0
    for n in nodes:
        want = dry_run(I, int(n))
        assert bool(out["ok"][n]) == (want is not None), (n, want)
        if want is None:
            continue
        hits += 1
        vic, keys = want
        o = int(I["rt_off"][n])
        assert int(out["nv"][n]) == len(vic), n
        assert list(out["victims"][o:o + len(vic)]) == vic, (n, vic)
        assert tuple(int(out["key"][k * N + n]) for k in range(4)) == keys, (n, keys)
    return hits


def splitmix64(x):
    m = (1 << 64) - 1
    z = (x + 0x9E3779B97F4A7C15) & m
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def select(pred, ok, keys, seed_k, pct, min_abs, max_abs):
    """findCandidates' single-worker reading + SelectCandidate -> (winner node or -1, P); keys [4][N]."""
    nodes = np.flatnonzero(pred)
    P = len(nodes)
    if P == 0:
        return -1, 0
    off = splitmix64(seed_k) % P
    numc = P * pct // 100 if pct >= 0 else -((-P * pct) // 100)  # Go's truncating division
    numc = max(numc, min_abs)
    numc = min(numc, max_abs, P)
    order = [int(nodes[(off + i) % P]) for i in range(P)]
    cands = [n for n in order if ok[n]][:max(numc, 0)]
    if not cands:
        return -1, P
    c = np.array(cands)
    # lexsort: the last key is primary; larger scores win, then the earlier candidate
    idx = np.lexsort((np.arange(len(c)), -keys[3][c], -keys[2][c], -keys[1][c], -keys[0][c]))
    return int(c[idx[0]]), P
