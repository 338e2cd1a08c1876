"""The incremental commit kernel (k_commit_fast, volcano_b200/csrc/vc_commit_fast.cuh) on every path it takes, against
the CPU oracle's allocate() on the same session: decisions (task, node, kind, visit, fp64 score) bit-equal, visits, fit
errors and, under sampling, the lastProcessedNodeIndex the action leaves.

The kernel's shortcuts engage only at some shapes, so every case asserts, worked out in Python, the precondition that
puts it on its path:
  * the instance (plain / FUT / SOFT / FUT+SOFT / SAMP / SAMP+FUT) and the launch geometry (a mirror of
    choose_geometry for the incremental kernel): CTAs, nodes per CTA, block and node rows per thread;
  * run_max, the queue mirror (Q <= 64) and where the job heap lives (shared or global memory);
  * the run-length batches: with VC_PROF_OWNER the library prints the run commands of the cycle and the placements
    they covered ("runs: X publications covering Y placements"). `_mirror` restates the control warp's run rule on the
    oracle's decision stream and predicts X and Y exactly on sessions without a discarded statement (a discarded
    visit carries no operations, so its runs leave no trace in the stream)."""
import dataclasses
import re

import numpy as np
import pytest

from tests.test_gpu_backfill import _integral, _to_find
from volcano_b200 import abi

pytestmark = pytest.mark.gpu

RUN_MAX = 32        # lanes of the evaluator warp: the most placements one publication covers
FAST_MAXQ = 64      # queues mirrored in shared memory
HEAP_KEY_BYTES = 32
HEAP_SMEM_MAX = 96 * 1024
RUNS_RE = re.compile(r"runs: (\d+) publications covering (\d+) placements")


@pytest.fixture(scope="module")
def gpu():
    from volcano_b200 import engine
    engine.init(0)
    return engine


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- restatements of the library's choices (preconditions only) ------------------------------------------------
def _plugins(snap):
    """{plugin id: enabled flags} of the session's configuration."""
    c = snap.conf
    out = {}
    for i in range(c.n_plugins):
        out[c.plugins[i].plugin] = out.get(c.plugins[i].plugin, 0) | c.plugins[i].enabled
    return out


def _flags(snap):
    p = _plugins(snap)
    prop = p.get(abi.VC_PLUGIN_PROPORTION)
    return {
        "gang_ready": bool(p.get(abi.VC_PLUGIN_GANG, 0) & abi.VC_EN_JOB_READY),
        "share_on": bool(p.get(abi.VC_PLUGIN_DRF, 0) & abi.VC_EN_JOB_ORDER),
        "prop": prop is not None,
        "over_prop": bool((prop or 0) & abi.VC_EN_OVERUSED),
        "alloc_prop": bool((prop or 0) & abi.VC_EN_ALLOCATABLE),
        "qorder_prop": bool((prop or 0) & abi.VC_EN_QUEUE_ORDER),
        "nodeorder": abi.VC_PLUGIN_NODEORDER in p,
    }


def _fut(snap):
    return bool(snap.n_releasing.any() or snap.n_pipelined.any())


def _soft(snap):
    return _flags(snap)["nodeorder"] and snap.conf.w_taint_toleration != 0 and bool(snap.n_taint_soft.any())


def _instance(snap):
    if _to_find(snap) > 0:
        return "samp+fut" if _fut(snap) else "samp"
    return {(False, False): "plain", (True, False): "fut", (False, True): "soft", (True, True): "fut+soft"}[(_fut(snap), _soft(snap))]


def _geometry(snap, opts, sm):
    """choose_geometry for the incremental kernel on one GPU: 256 threads unless VC_COMMIT_THREADS, 128 nodes per CTA
    from 64 x 128 nodes on when the CTA count is not forced."""
    N = snap.N
    ctas = opts.get("VC_COMMIT_CTAS", 0) or sm
    block = 128
    if opts.get("VC_COMMIT_THREADS", 0):
        block = max(128, min(256, opts["VC_COMMIT_THREADS"] // 32 * 32))
    ctas = max(1, min(ctas, (N + 31) // 32))
    npc = max(32, (-(-N // ctas) + 31) // 32 * 32)
    if not opts.get("VC_COMMIT_CTAS", 0) and npc < 128 and N >= 64 * 128:
        npc = 128
    ctas = max(1, -(-N // npc))
    if npc > block:
        block = min(256, (npc + 31) // 32 * 32)
    if not opts.get("VC_COMMIT_THREADS", 0):
        block = 256
    return {"ctas": ctas, "npc": npc, "block": block, "rows": -(-npc // block)}


def _rows_integral(snap):
    """vch::runs_exact over the node rows and the pending tasks' requests."""
    if not _integral(snap.n_idle, snap.n_used, snap.n_releasing, snap.n_pipelined, snap.n_k8s_requested,
                     snap.n_k8s_nonzero_requested, snap.t_resreq, snap.t_k8s_req, snap.t_k8s_nonzero_req):
        return False
    for rows, req in (((snap.n_idle, snap.n_used), snap.t_resreq), ((snap.n_k8s_requested,), snap.t_k8s_req),
                      ((snap.n_k8s_nonzero_requested[:2],), snap.t_k8s_nonzero_req[:2])):
        mrow = np.max([np.abs(r).max(axis=1) for r in rows], axis=0)
        if not (mrow + 32.0 * np.abs(req).max(axis=1) < 9.0e15).all():
            return False
    return True


def _run_max(snap, opts, geo):
    if _to_find(snap) > 0 or opts.get("VC_COMMIT_NORUN") or not _rows_integral(snap):
        return 1
    cap = min(RUN_MAX, 2 * (geo["block"] // 32 - 1))
    return max(1, min(opts.get("VC_RUN_MAX") or RUN_MAX, cap))


def _heap_total(snap):
    """Re-pushable jobs (allocate.go:334-336): Ready with a task left is possible, or any second task without gang."""
    scope = np.bincount(snap.t_job, minlength=snap.J)
    if _flags(snap)["gang_ready"]:
        return int((snap.j_ready_num + snap.j_pending_besteffort + scope > snap.j_min_available).sum())
    return int((scope >= 2).sum())


def _heap_in_global(snap):
    return _heap_total(snap) * HEAP_KEY_BYTES > HEAP_SMEM_MAX


def _groups(snap):
    """(class, has-bits, request rows) group of every pending task."""
    def cols(a):
        return np.ascontiguousarray(np.asarray(a, np.float64).T).view(np.int64)
    key = np.concatenate([snap.t_klass.astype(np.int64)[:, None], snap.t_req_has.astype(np.int64)[:, None],
                          cols(snap.t_resreq), cols(snap.t_k8s_req), cols(snap.t_k8s_nonzero_req[:2])], axis=1)
    return np.unique(key, axis=0, return_inverse=True)[1].ravel()


# ---- the run rule on the oracle's decision stream --------------------------------------------------------------
def _mirror(snap, ref, run_max, des):
    """The control warp's run rule (vc_commit_fast.cuh, "run length") replayed on the oracle's decisions.

    A run starts at every allocation of a job that no earlier run covers. Its length run_L comes from the state before
    it: placements until ssn.JobReady (role minima included: another role short never makes the job Ready), or, for a
    Ready job popped from the heap, RUN_MAX further one-task visits when nothing can come between them (no drf share
    in JobOrderFn, the queue mirrored, proportion's overused off, the queue popped again: no other queue left under
    hdrf or proportion's queue order); then the same group and role
    in the job's task order, run_max, and proportion's queueAllocatable per dimension. The run covers the placement and
    the following allocations of the job's next tasks on the same node, up to run_L.
    -> {"X", "Y", "runs": [(decision index, run_L, covered, cross-visit)], "exact"}"""
    f = _flags(snap)
    dec, vis, fe = ref
    grp = _groups(snap)
    ready = snap.j_ready_num.astype(np.int64).copy()
    occ = snap.r_occupied.astype(np.int64).copy()
    qalloc = snap.q_allocated.copy()
    minav, pbe, tmin = snap.j_min_available, snap.j_pending_besteffort, snap.j_task_min_total
    in_min = (snap.r_flags & abi.VC_ROLE_IN_MIN_MAP) != 0
    roff = snap.j_role_off
    failed = np.bincount(snap.t_job[fe], minlength=snap.J) if len(fe) else np.zeros(snap.J, np.int64)
    # the job's task order: its decided tasks in the order of the stream, then the tasks never placed
    seq = [[] for _ in range(snap.J)]
    for t in dec["task"]:
        seq[snap.t_job[t]].append(int(t))
    pos = {t: i for s in seq for i, t in enumerate(s)}
    placed = np.zeros(snap.T, bool)
    placed[dec["task"]] = True
    rest = [[] for _ in range(snap.J)]
    for t in np.flatnonzero(~placed):
        rest[snap.t_job[t]].append(int(t))
    jq = snap.j_queue
    last_visit_of_q = np.full(snap.Q, -1)
    for v, r in enumerate(vis):
        last_visit_of_q[jq[r["job"]]] = v
    hd = snap.hdrf() is not None
    seen = set()
    op_visit = np.repeat(np.arange(len(vis)), vis["n_ops"])
    assert len(op_visit) == len(dec)
    X = Y = 0
    runs, exact, covered = [], True, 0
    for k in range(len(dec)):
        v = op_visit[k]
        j = int(vis["job"][v])
        from_heap = j in seen
        t, node, kind = int(dec["task"][k]), int(dec["node"][k]), int(dec["kind"][k])
        q = int(jq[j])
        rl = int(snap.t_role[t])
        if covered == 0 and kind == abi.VC_OP_ALLOCATE and run_max > 1:
            need = 0
            if f["gang_ready"]:
                need = int(minav[j] - pbe[j] - ready[j])
                roles = range(roff[j], roff[j + 1])
                if any(in_min[r] for r in roles) and not minav[j] < tmin[j]:
                    short = [r for r in roles if in_min[r] and occ[r] < snap.r_min[r]]
                    need_rl = int(snap.r_min[rl] - occ[rl]) if rl in short else 0
                    need = RUN_MAX + 1 if any(r != rl for r in short) else max(need, need_rl)
            lim, vrun = 0, False
            if need > 1:
                lim = need
            elif need <= 0 and from_heap and not f["share_on"] and snap.Q <= FAST_MAXQ and not (f["over_prop"] and f["prop"]):
                # another queue still to be served: under hdrf it is in the queue heap, under proportion's queue order
                # it may be popped first; either way the job's queue is not popped again for sure
                others = sum(1 for q2 in range(snap.Q) if q2 != q and last_visit_of_q[q2] > v)
                if not (hd or f["qorder_prop"]) or others == 0:
                    lim, vrun = RUN_MAX, True
            run_L = 1
            if lim > 1:
                n_same = 0  # the job's next tasks of this group and role
                for t2 in seq[j][pos[t] + 1:] + rest[j]:
                    if grp[t2] != grp[t] or snap.t_role[t2] != rl:
                        exact = exact and not (rest[j] and pos[t] + 1 + n_same >= len(seq[j]))
                        break
                    n_same += 1
                if failed[j]:
                    exact = False  # where the job's fit errors sit in its task order is not in the stream
                run_L = min(1 + min(n_same, 32), lim, run_max)
            if run_L > 1 and f["alloc_prop"] and f["prop"]:
                run_L = min(run_L, _gate(snap, t, qalloc[:, q], des[:, q], run_L))
            if run_L > 1:
                follow = 0  # the next allocations of this job, same group, same node
                for k2 in range(k + 1, len(dec)):
                    v2 = op_visit[k2]
                    if vrun and (vis["job"][v2] != j or vis["n_ops"][v2] != 1):
                        break
                    if not vrun and v2 != v:
                        break
                    t2 = int(dec["task"][k2])
                    if dec["node"][k2] != node or dec["kind"][k2] != abi.VC_OP_ALLOCATE or grp[t2] != grp[t] or snap.t_role[t2] != rl:
                        break
                    follow += 1
                m = 1 + min(run_L - 1, follow)
                X += 1
                Y += m
                runs.append((k, run_L, m, vrun))
                covered = m
        if covered:
            covered -= 1
        seen.add(j)
        if kind == abi.VC_OP_ALLOCATE:
            ready[j] += 1
            occ[rl] += 1
        has = int(snap.t_req_has[t])
        for d in range(snap.R):
            if d < 2 or has & (1 << d):
                qalloc[d, q] += snap.t_resreq[d, t]
    return {"X": X, "Y": Y, "runs": runs, "exact": exact}


def _gate(snap, t, qalloc, des, run_L):
    """proportion's queueAllocatable for the placements after the first, one dimension at a time: placement c + 1 passes
    while allocated + request <= deserved (equality allowed); cpu and memory always, scalars the task requests, never
    pods."""
    has = int(snap.t_req_has[t]) & ~3
    out = run_L
    for d in range(snap.R):
        req = snap.t_resreq[d, t]
        if not (d < 2 or (has & (1 << d) and d != snap.pods_dim)) or req <= 0:
            continue
        qa, cnt = qalloc[d] + req, 1
        while cnt < run_L and not qa + req > des[d]:
            qa += req
            cnt += 1
        out = min(out, cnt)
    return out


# ---- running both sides --------------------------------------------------------------------------------------------
def _oracle(snap, threads=4):
    """The CPU oracle's allocate(); the hdrf oracle on sessions with drf's enableHierarchy."""
    from oracle import pyoracle
    from oracle.pyoracle import OracleSession
    if snap.hdrf() is not None:
        from tests import hdrf_common
        o = hdrf_common.oracle_for(snap, snap.api_queues)
        return {"alloc": o.allocate(), "last": -1, "des": np.zeros((snap.R, snap.Q))}
    o = OracleSession(snap, threads=threads)
    des, _ = o.queue_deserved()
    res = o.allocate()
    last = int(pyoracle.lib().vco_last_processed_node_index(o.h))
    o.close()
    return {"alloc": res, "last": last, "des": des}


def _library(gpu, capfd, snap, opts=None):
    opts = dict(opts or {}, VC_PROF_OWNER=1)
    capfd.readouterr()
    for k, v in opts.items():
        gpu.debug_option(k, v)
    try:
        e = gpu.Engine(snap)
        e.upload()
        res = e.allocate()
        e.close()
    finally:
        for k in opts:
            gpu.debug_option(k, 0)
    m = RUNS_RE.findall(capfd.readouterr().err)
    assert len(m) == 1, m
    res.runs = tuple(int(x) for x in m[0])
    return res


def _same(got, ref, samp):
    dec, vis, fe = ref["alloc"]
    assert np.array_equal(got.visits, vis), "visits differ"
    for f in ("task", "node", "kind", "visit"):
        bad = np.flatnonzero(got.decisions[f] != dec[f]) if len(got.decisions) == len(dec) else [-1]
        assert len(got.decisions) == len(dec) and not len(bad), f"decision {f} differs from index {bad[0]}"
    assert np.array_equal(got.decisions["score"].view(np.int64), dec["score"].view(np.int64)), "fp64 scores differ"
    assert np.array_equal(got.fit_errors, fe), "fit errors differ"
    if samp:
        assert got.stats["last_processed_node_index"] == ref["last"]


def _check(gpu, capfd, snap, ref, sm, opts=None, instance=None, exact=True):
    """Parity, the instance, and the run counts against the mirror; exact=None: exact whenever no visit was discarded
    and the mirror is exact, otherwise runs engaged (X > 0, Y > X) where run_max allows them. -> (result, mirror)"""
    opts = dict(opts or {})
    geo = _geometry(snap, opts, sm)
    if instance is not None:
        assert _instance(snap) == instance
    rm = _run_max(snap, opts, geo)
    mir = _mirror(snap, ref["alloc"], rm, ref["des"])
    got = _library(gpu, capfd, snap, opts)
    assert got.stats["commit_kernel"] == 1, got.stats  # VC_KERNEL_INCREMENTAL
    _same(got, ref, _to_find(snap) > 0)
    if rm == 1:
        assert got.runs == (0, 0)
    if exact is None:
        exact = not (ref["alloc"][1]["outcome"] == abi.VC_VISIT_DISCARD).any() and mir["exact"]
        if not exact and rm > 1:
            assert got.runs[0] > 0 and got.runs[1] > got.runs[0], got.runs
    if exact:
        assert (ref["alloc"][1]["outcome"] == abi.VC_VISIT_DISCARD).sum() == 0
        assert mir["exact"]
        assert got.runs == (mir["X"], mir["Y"]), (got.runs, mir["X"], mir["Y"], mir["runs"][:20])
    return got, mir


# ---- small hand-built sessions -------------------------------------------------------------------------------------
BINPACK = {"binpack.weight": 10, "binpack.cpu": 5, "binpack.memory": 1}


def _tiers(plugins):
    """'+'-separated plugins at their defaults; "hdrf" is drf with enableHierarchy and its queue order only (no share in
    JobOrderFn)."""
    from volcano_b200.snapshot import PluginOption

    def opt(n):
        if n == "hdrf":
            return PluginOption.make("drf", EnabledHierarchy=True, EnabledQueueOrder=True)
        return PluginOption.defaults(n, BINPACK if n == "binpack" else None)
    names = plugins.split("+")
    t1 = [opt(n) for n in names if n in ("priority", "gang")]
    t2 = [opt(n) for n in names if n not in ("priority", "gang")]
    return [t for t in (t1, t2) if t]


def _cluster(jobs, nodes=((64, 256, 110),) * 2, queues=(("q", 1, None, 0),), plugins="priority+gang+predicates+binpack",
             running=(), drop=(), **conf_kw):
    """jobs: dicts (name, n, min, cpu, mem in Gi, queue, gpu, roles [(role, count, priority or one per pod[, cpu])],
    task_min, selector); nodes: (cpu, memory Gi, pods[, labels[, gpu]]); queues: (name, weight, capability,
    priority[, hdrf path, hdrf weights]); running: (job, node, role, cpu, deleting) pods already placed; drop: (plugin,
    VC_EN_* flags) switched off after the defaults."""
    from volcano_b200 import api
    from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildResourceList
    from volcano_b200.uthelper import TestCommonStruct
    ns = []
    for i, nd in enumerate(nodes):
        extra = [("pods", str(nd[2]))] + ([("nvidia.com/gpu", str(nd[4]))] if len(nd) > 4 else [])
        ns.append(BuildNode(f"n{i:04d}", BuildResourceList(str(nd[0]), f"{nd[1]}Gi", *extra), nd[3] if len(nd) > 3 else {}))
    pods, pgs = [], []
    for jb in jobs:
        roles = jb.get("roles") or [("w", jb["n"], None)]
        for role, cnt, prio, *cpu in roles:
            for i in range(cnt):
                req = BuildResourceList(str(cpu[0] if cpu else jb.get("cpu", 1)), f"{jb.get('mem', 1)}Gi",
                                        *([("nvidia.com/gpu", str(jb["gpu"]))] if jb.get("gpu") else []))
                p = BuildPod("ns", f"{jb['name']}-{role}-{i}", "", "Pending", req, jb["name"],
                             {api.TASK_SPEC_KEY: role}, jb.get("selector"))
                p.priority = prio[i] if isinstance(prio, (list, tuple)) else prio
                pods.append(p)
        pg = BuildPodGroup(jb["name"], "ns", jb.get("queue", "q"), jb["min"], jb.get("task_min"))
        pg.priority = jb.get("prio", 0)
        pgs.append(pg)
    for i, (job, node, role, cpu, deleting) in enumerate(running):
        p = BuildPod("ns", f"{job}-{role}-r{i}", f"n{node:04d}", "Running", BuildResourceList(str(cpu), "1Gi"), job,
                     {api.TASK_SPEC_KEY: role})
        p.deleting = deleting
        pods.append(p)
    qs = []
    for name, w, cap, prio, *hd in queues:
        q = api.BuildQueue(name, w, cap)
        q.priority = prio
        if hd:
            q.hierarchy, q.weights = hd
        qs.append(q)
    tc = TestCommonStruct(Name="commit-paths", Nodes=ns, Pods=pods, PodGroups=pgs, Queues=qs)
    snap = tc.RegisterSession(_tiers(plugins), **conf_kw)
    snap.api_queues = qs  # the hdrf oracle takes the queues' annotations
    for name, flags in drop:
        pid = abi.PLUGIN_IDS[name]
        for i in range(snap.conf.n_plugins):
            if snap.conf.plugins[i].plugin == pid:
                snap.conf.plugins[i].enabled &= ~flags
    return snap


def _gang(n, mn, **kw):
    return dict(name=kw.pop("name", "j"), n=n, min=mn, **kw)


def _runs_of(mir):
    return [(L, m, bool(x)) for _, L, m, x in mir["runs"]]


# ---- 1. run caps ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [2, 13, 14, 15])
def test_need_to_ready_caps_the_run(L, gpu, capfd, sm_count):
    """One gang of L + 4 one-cpu pods with minMember L on two nodes under binpack: the first visit places L pods on one
    node in runs cut where ssn.JobReady turns true (and at run_max 14: 15 = 14 + 1), then the Ready job's last four
    pods come one visit each, folded into one cross-visit run."""
    snap = _cluster([_gang(L + 4, L)])
    ref = _oracle(snap)
    geo = _geometry(snap, {}, sm_count)
    assert geo == {"ctas": 1, "npc": 32, "block": 256, "rows": 1} and _run_max(snap, {}, geo) == 14
    assert _heap_total(snap) == 1 and not _heap_in_global(snap)
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="plain")
    assert _runs_of(mir) == [(min(L, 14), min(L, 14), False), (4, 4, True)], _runs_of(mir)
    assert mir["X"] > 0 and mir["Y"] > mir["X"]


RUN_END_CASES = {
    # a Ready job's cross-visit run ends at its last task (n_same)
    "job_last_task": (lambda: _cluster([_gang(9, 3)]), [(3, 3, False), (6, 6, True)]),
    # the node's pod cap (6 pods) ends the run; the other (larger, so binpack's second choice) node takes the rest
    "pod_cap": (lambda: _cluster([_gang(10, 10)], nodes=((64, 256, 6), (128, 256, 110))), [(10, 6, False), (4, 4, False)]),
    # cpu runs out on the node after 4 pods (4.5 cpu)
    "resource_out": (lambda: _cluster([_gang(10, 10)], nodes=(("4500m", 256, 110), (32, 256, 110))),
                     [(10, 4, False), (6, 6, False)]),
    # leastrequested + balanced spread the pods: the node loses the arg-max after every placement (runs of one)
    "argmax_lost": (lambda: _cluster([_gang(12, 12)], nodes=((64, 256, 110),) * 4, plugins="priority+gang+predicates+nodeorder"),
                    [(12 - i, 1, False) for i in range(11)]),
}


@pytest.mark.parametrize("name", sorted(RUN_END_CASES))
def test_run_ends(name, gpu, capfd, sm_count):
    build, want = RUN_END_CASES[name]
    snap = build()
    ref = _oracle(snap)
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="plain")
    assert _runs_of(mir) == want, _runs_of(mir)


ROLE_CASES = {
    # roles a (priority 2, first in the task order) and b: minMember 4, minima a 2 / b 2. At a's first pod b is short:
    # the run covers all six a pods (a's own minimum does not end it); b's first pod: b short by 2, a run of 2
    "other_short": (dict(roles=[("a", 6, 2), ("b", 3, 1)], task_min={"a": 2, "b": 2}, mn=4), (),
                    [(6, 6, False), (2, 2, False)]),
    # two b pods already run (ready 2): minMember 5, minimum a 4: need to Ready is 3, a's own shortfall 4 decides
    "this_short": (dict(roles=[("a", 6, 2)], task_min={"a": 4}, mn=5), (("j", 1, "b", 1, False),) * 2,
                   [(4, 4, False), (2, 2, True)]),
    # both: a short by 4 and b short by 2 at the start (six a, three b, minMember 6)
    "both_short": (dict(roles=[("a", 6, 2), ("b", 3, 1)], task_min={"a": 4, "b": 2}, mn=6), (),
                   [(6, 6, False), (2, 2, False)]),
}


@pytest.mark.parametrize("name", sorted(ROLE_CASES))
def test_role_minima(name, gpu, capfd, sm_count):
    kw, running, want = ROLE_CASES[name]
    kw = dict(kw)
    mn = kw.pop("mn")
    n = sum(c for _, c, _ in kw["roles"])
    snap = _cluster([_gang(n, mn, **kw)], running=running)
    assert (snap.r_flags & abi.VC_ROLE_IN_MIN_MAP).any() and snap.j_task_min_total[0] <= snap.j_min_available[0]
    ref = _oracle(snap)
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="plain")
    assert _runs_of(mir) == want, _runs_of(mir)


PROP_CASES = {
    # capability caps deserved: cpu binds at 5 (memory at 8 would not)
    "cpu_binds": ({"cpu": "5", "memory": "8Gi"}, 5),
    # memory binds at 5 (cpu at 8 would not)
    "memory_binds": ({"cpu": "8", "memory": "5Gi"}, 5),
    # allocated + request == deserved is allowed: 5000m admits the fifth pod, 4999m refuses it
    "equal_allowed": ({"cpu": "5000m", "memory": "64Gi"}, 5),
    "one_unit_over": ({"cpu": "4999m", "memory": "64Gi"}, 4),
    # a requested scalar binds (three gpus)
    "gpu_binds": ({"cpu": "64", "memory": "64Gi", "nvidia.com/gpu": "3"}, 3),
    # pods is never counted: a pods capability of 2 does not cut the run
    "pods_not_counted": ({"cpu": "6", "memory": "64Gi", "pods": "2"}, 6),
}


@pytest.mark.parametrize("name", sorted(PROP_CASES))
def test_proportion_gate(name, gpu, capfd, sm_count):
    """A Ready job (minMember 1, twelve pods) in a queue whose capability caps deserved: after the first visit the
    cross-visit run is cut by the queueAllocatable simulation partway, and the oracle refuses the pod after it."""
    cap, k = PROP_CASES[name]
    gpu_req = 1 if "gpu" in name else None
    snap = _cluster([_gang(12, 1, gpu=gpu_req)], nodes=((64, 256, 110, {}, 16),) * 2, queues=(("q", 1, cap, 0),),
                    plugins="priority+gang+predicates+proportion+binpack", drop=(("proportion", abi.VC_EN_OVERUSED),))
    f = _flags(snap)
    assert f["alloc_prop"] and not f["over_prop"] and f["qorder_prop"]
    ref = _oracle(snap)
    dec = ref["alloc"][0]
    assert len(dec) == k, len(dec)
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="plain")
    assert _runs_of(mir) == [(k - 1, k - 1, True)], _runs_of(mir)
    des, d = ref["des"][:, 0], snap.pods_dim
    if name == "equal_allowed":
        assert des[0] == 5000.0 == k * snap.t_resreq[0, 0]
    if name == "pods_not_counted":
        assert des[d] < k


# ---- 2. cross-visit runs and where they are off --------------------------------------------------------------------
def _ready_job_session(plugins, queues=(("q", 1, None, 0),), drop=(), extra_jobs=()):
    """A Ready job (minMember 2 of twelve pods) in queue q: the first visit places 2, each later visit one."""
    return _cluster([_gang(12, 2)] + list(extra_jobs), queues=queues, plugins=plugins, drop=drop)


VRUN_CASES = {
    "engaged": (lambda: _ready_job_session("priority+gang+predicates+binpack"), True),
    # drf's share in JobOrderFn: the job's key moves with every placement
    "drf_job_order": (lambda: _ready_job_session("priority+gang+drf+predicates+binpack"), False),
    # proportion's overused check between the visits
    "overused": (lambda: _ready_job_session("priority+gang+predicates+proportion+binpack"), False),
    # proportion's queue order with another active queue (a lower-priority queue served last)
    "multi_queue_order": (lambda: _ready_job_session(
        "priority+gang+predicates+proportion+binpack", queues=(("q", 1, None, 1), ("low", 1, None, 0)),
        drop=(("proportion", abi.VC_EN_OVERUSED),), extra_jobs=[_gang(2, 2, name="k", queue="low")]), False),
    # 65 queues: no shared-memory mirror of the queue states
    "q65": (lambda: _ready_job_session("priority+gang+predicates+binpack",
                                       queues=tuple((f"q{i}" if i else "q", 1, None, 0) for i in range(65))), False),
    # hdrf with the job's queue alone in the tree: the queue heap is otherwise empty, the queue is popped again
    "hdrf_alone": (lambda: _ready_job_session("priority+gang+hdrf+predicates+binpack",
                                              queues=(("q", 1, None, 0, "root/a", "1/1"),)), True),
    # hdrf with a second queue that outlasts the job: it stays in the queue heap, so no visit is folded. Its job
    # alternates two requests in its task order (no run of its own either)
    "hdrf_busy": (lambda: _ready_job_session(
        "priority+gang+hdrf+predicates+binpack", queues=(("q", 1, None, 0, "root/a", "1/1"), ("b", 1, None, 0, "root/b", "1/1")),
        extra_jobs=[_gang(24, 1, name="k", queue="b", roles=[("x", 12, list(range(48, 0, -4)), 1),
                                                            ("y", 12, list(range(46, 0, -4)), 2)])]), False),
}


@pytest.mark.parametrize("name", sorted(VRUN_CASES))
def test_cross_visit_runs(name, gpu, capfd, sm_count):
    build, engaged = VRUN_CASES[name]
    snap = build()
    ref = _oracle(snap)
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="plain")
    cross = [r for r in _runs_of(mir) if r[2]]
    if engaged:
        assert cross == [(10, 10, True)], _runs_of(mir)
    else:
        assert not cross and mir["X"] >= 1, _runs_of(mir)  # the in-visit run of the first visit only
    if name == "q65":
        assert snap.Q > FAST_MAXQ
    if name.startswith("hdrf"):
        assert snap.hdrf() is not None and not _flags(snap)["share_on"]
    if name == "hdrf_busy":  # the other queue is served after the job's last visit
        dec, vis, _ = ref["alloc"]
        jobs = list(vis["job"])
        assert max(i for i, j in enumerate(jobs) if j == 0) < max(i for i, j in enumerate(jobs) if j == 1)
        assert jobs.count(1) > 12 and mir["X"] == 1


# ---- 3. single candidate -------------------------------------------------------------------------------------------
def test_single_candidate_run(gpu, capfd, sm_count):
    """A gang pinned by a selector to one of four nodes: one candidate at every placement (score 0.0 without a score
    log read)."""
    nodes = [(64, 256, 110, {"pin": "yes" if i == 2 else "no"}) for i in range(4)]
    snap = _cluster([_gang(8, 8, selector={"pin": "yes"})], nodes=nodes)
    ref = _oracle(snap)
    dec = ref["alloc"][0]
    assert len(dec) == 8 and (dec["node"] == 2).all() and (dec["score"] == 0.0).all()
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="plain")
    assert _runs_of(mir) == [(8, 8, False)]


def test_single_candidate_fut_boundary(gpu, capfd, sm_count):
    """FUT: the pinned node has idle room for three pods and releasing room for three more. The run stops where the
    row leaves the idle category; the next placement is a pipeline on the same node."""
    nodes = [(11 if i == 1 else 8, 256, 110, {"pin": "yes" if i == 1 else "no"}) for i in range(3)]
    running = [("old", 1, "w", 5, False), ("old", 1, "w", 3, True)]  # 5 cpu used, 3 releasing: 3 idle
    snap = _cluster([_gang(6, 6, selector={"pin": "yes"}), _gang(0, 1, name="old")], nodes=nodes, running=running)
    ref = _oracle(snap)
    dec = ref["alloc"][0]
    assert list(dec["kind"]) == [abi.VC_OP_ALLOCATE] * 3 + [abi.VC_OP_PIPELINE] * 3 and (dec["node"] == 1).all()
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="fut")
    assert _runs_of(mir) == [(6, 3, False)]


# ---- 4. run length by block size -----------------------------------------------------------------------------------
RUN_OPTS = [({}, 14), ({"VC_COMMIT_THREADS": 128}, 6), ({"VC_COMMIT_THREADS": 256}, 14), ({"VC_RUN_MAX": 1}, 1),
            ({"VC_RUN_MAX": 2}, 2), ({"VC_RUN_MAX": 13}, 13), ({"VC_COMMIT_NORUN": 1}, 1)]


@pytest.mark.parametrize("opts,rm", RUN_OPTS, ids=["default", "t128", "t256", "max1", "max2", "max13", "norun"])
def test_run_max(opts, rm, gpu, capfd, sm_count):
    """A gang of 40 (minMember 30) and a Ready job of 20 (minMember 2) on binpack: runs cut at run_max in both kinds."""
    snap = _cluster([_gang(40, 30), _gang(20, 2, name="r")], nodes=((128, 512, 250),) * 2)
    ref = _oracle(snap)
    assert _run_max(snap, opts, _geometry(snap, opts, sm_count)) == rm
    _, mir = _check(gpu, capfd, snap, ref, sm_count, opts, instance="plain")
    if rm > 1:
        assert max(L for L, _, _ in _runs_of(mir)) == rm and any(x for _, _, x in _runs_of(mir))
        assert mir["Y"] > mir["X"] > 0


# ---- 5. state outside shared memory --------------------------------------------------------------------------------
def _synth(base, **changes):
    from volcano_b200.synth import CONFIGS, make_snapshot
    return make_snapshot(dataclasses.replace(CONFIGS[base], name=f"{base}-paths", **changes))


def _exact_or_runs(gpu, capfd, snap, ref, sm, opts=None, instance=None):
    return _check(gpu, capfd, snap, ref, sm, opts, instance, exact=None)


@pytest.mark.parametrize("Q", [65, 80])
def test_queues_without_mirror(Q, gpu, capfd, sm_count):
    snap = _synth("small", n_queues=Q, n_tasks=3000)
    assert snap.Q > FAST_MAXQ
    ref = _oracle(snap)
    _exact_or_runs(gpu, capfd, snap, ref, sm_count, instance="plain")


def test_global_memory_heap(gpu, capfd, sm_count):
    """3 100 jobs of three pods with minMember 1: every job can come back, 3 100 x 32 B of heap is over 96 KiB."""
    jobs = [_gang(3, 1, name=f"j{i}") for i in range(3100)]
    snap = _cluster(jobs, nodes=((250, 512, 250),) * 40)
    assert _heap_total(snap) == 3100 and _heap_in_global(snap)
    ref = _oracle(snap)
    _, mir = _check(gpu, capfd, snap, ref, sm_count, instance="plain")
    assert any(x for _, _, x in _runs_of(mir))


def test_mid_size_rounds_to_128_nodes(gpu, capfd, sm_count):
    """10 000 nodes on one GPU: the node axis over every SM would give fewer than 128 nodes per CTA (96 on 132 SMs); the
    incremental kernel takes 128 (79 CTAs)."""
    snap = _synth("cfg2", n_tasks=6000)
    geo = _geometry(snap, {}, sm_count)
    assert (-(-snap.N // sm_count) + 31) // 32 * 32 < 128 and geo["npc"] == 128 and geo["ctas"] == -(-snap.N // 128), geo
    ref = _oracle(snap, threads=8)
    _exact_or_runs(gpu, capfd, snap, ref, sm_count, instance="plain")


def test_40k_nodes_two_rows(gpu, capfd, sm_count):
    snap = _synth("cfg2", n_nodes=40_000, n_tasks=20_000)
    geo = _geometry(snap, {}, sm_count)
    assert geo["rows"] == 2 and geo["npc"] > 256, geo
    ref = _oracle(snap, threads=8)
    _exact_or_runs(gpu, capfd, snap, ref, sm_count, instance="plain")


CTAS_CASES = [
    ("plain_1cta", "small", dict(n_nodes=500, n_queues=1, plugins="priority+gang+predicates+nodeorder+binpack"), 1, "plain"),
    ("plain_2cta", "small", dict(n_nodes=1000, n_queues=1, plugins="priority+gang+predicates+nodeorder+binpack"), 2, "plain"),
    ("fut_2cta", "mid_fut", dict(n_nodes=800, n_tasks=4000), 2, "fut"),
    ("soft_2cta", "small_soft", dict(n_nodes=1000, n_tasks=4000), 2, "soft"),
]


@pytest.mark.parametrize("name,base,kw,ctas,inst", CTAS_CASES, ids=[c[0] for c in CTAS_CASES])
def test_few_ctas_several_rows(name, base, kw, ctas, inst, gpu, capfd, sm_count):
    snap = _synth(base, **kw)
    opts = {"VC_COMMIT_CTAS": ctas}
    geo = _geometry(snap, opts, sm_count)
    assert geo["ctas"] == ctas and geo["rows"] >= 2, geo
    ref = _oracle(snap)
    _exact_or_runs(gpu, capfd, snap, ref, sm_count, opts, instance=inst)


def test_four_rows_one_cta(gpu, capfd, sm_count):
    """1 000 nodes on one CTA: 1 024 node slots, four rows of 256 threads."""
    snap = _wide(1000)
    opts = {"VC_COMMIT_CTAS": 1}
    assert _geometry(snap, opts, sm_count) == {"ctas": 1, "npc": 1024, "block": 256, "rows": 4}
    ref = _oracle(snap)
    _check(gpu, capfd, snap, ref, sm_count, opts, instance="plain")


def test_cfg4_flat_sampled_replay(gpu, sm_count):
    """cfg4_flat at full size (50 000 nodes x 1 000 000 pods, 16 queues, drf + proportion): 384-node slices, the heap in
    global memory. The GPU's decisions are replayed through the oracle and every 100th is re-derived."""
    import os
    from oracle.pyoracle import OracleSession
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot("cfg4_flat")
    geo = _geometry(snap, {}, sm_count)
    npc = (-(-snap.N // sm_count) + 31) // 32 * 32  # 384 on 132 SMs
    assert geo["npc"] == npc > 256 and geo["rows"] == 2 and _heap_in_global(snap) and _instance(snap) == "plain", geo
    res = gpu.gpu_engine(snap)
    assert res.stats["commit_kernel"] == 1 and len(res.decisions) > 500_000
    o = OracleSession(snap, threads=max(1, min(16, os.cpu_count() or 1)))
    bad, first, checked = o.replay_check(res.decisions, res.visits, 100, 41)
    o.close()
    assert checked >= len(res.decisions) // 100 - 1
    assert bad == 0, f"{bad} of {checked} sampled decisions differ, first at index {first}"


# ---- 6. SAMP windows -----------------------------------------------------------------------------------------------
SAMPLING = [
    # name, base, (pct, min nodes, start), options
    ("window_in_one_cta", "small", (1, 5, 3), {}),
    ("window_over_ctas", "small", (15, 20, 40), {}),
    ("start_near_n", "small", (5, 30, 690), {}),
    ("start_past_n", "small", (10, 20, 700 + 123), {}),
    ("fewer_feasible", "small", (20, 10, 100), {}),
    ("fut", "tiny_fut", (40, 8, 5), {}),
    ("four_rows", "small", (10, 20, 50), {"VC_COMMIT_CTAS": 1}),
]


def _wide(n_nodes, **conf_kw):
    """Three resource dimensions on n_nodes nodes: 1 000+ node slots of one CTA fit its shared memory."""
    jobs = [_gang(8, 4, name=f"j{i}", cpu=1 + i % 2) for i in range(60)]
    return _cluster(jobs, nodes=[(16 + 16 * (i % 3), 64, 110) for i in range(n_nodes)], **conf_kw)


def _samp_snapshot(name, base, args):
    pct, mn, start = args
    if name == "four_rows":
        return _wide(1000, percentage_nodes_to_find=pct, min_nodes_to_find=mn, last_processed_node_index=start)
    snap = _synth(base)
    if name == "fewer_feasible":  # every pod in one class that selects one zone (~1/16 of the nodes)
        zone = snap.C - 1
        snap.c_selector[zone] = 0
        snap.c_selector[zone, 0] = np.uint64(1) << np.uint64(5)
        snap.t_klass[:] = zone
    snap.conf.percentage_nodes_to_find, snap.conf.min_nodes_to_find, snap.conf.last_processed_node_index = pct, mn, start
    return snap


@pytest.mark.parametrize("name,base,args,opts", SAMPLING, ids=[s[0] for s in SAMPLING])
def test_sampling_windows(name, base, args, opts, gpu, capfd, sm_count):
    snap = _samp_snapshot(name, base, args)
    geo = _geometry(snap, opts, sm_count)
    tf, N, npc = _to_find(snap), snap.N, geo["npc"]
    start = args[2] % N
    assert tf > 0
    if name == "window_in_one_cta":
        assert start % npc + tf < npc
    if name == "window_over_ctas":
        assert tf > 2 * npc
    if name == "start_near_n":
        assert start // npc == geo["ctas"] - 1 and start + tf > N
    if name == "start_past_n":
        assert args[2] >= N
    if name == "fewer_feasible":
        sel = snap.c_selector[snap.C - 1, 0]
        assert ((snap.n_label_bits[0] & sel) == sel).sum() < tf
    if name == "four_rows":
        assert geo == {"ctas": 1, "npc": 1024, "block": 256, "rows": 4}
    ref = _oracle(snap, threads=1)
    dec, vis, fe = ref["alloc"]
    assert len(dec) > 0
    # steps of one group in a row (the window published ahead is taken) and group switches (it is dropped)
    g = _groups(snap)[dec["task"]]
    assert (g[1:] == g[:-1]).any() and (g[1:] != g[:-1]).any()
    if name == "fewer_feasible":  # and the window dropped after a discard or a fit error, with the same group next
        vg = _groups(snap)[[int(np.flatnonzero(snap.t_job == j)[0]) for j in vis["job"]]]  # one group per synthetic job
        same_next = np.append(vg[1:] == vg[:-1], False)
        assert (same_next & (vis["outcome"] == abi.VC_VISIT_DISCARD)).any()
        failing = np.isin(vis["job"], snap.t_job[fe])
        assert (same_next & failing & (vis["outcome"] != abi.VC_VISIT_DISCARD)).any()
    _check(gpu, capfd, snap, ref, sm_count, opts, instance="samp+fut" if name == "fut" else "samp", exact=False)


def test_sampling_five_rows_refused(gpu, sm_count):
    """1 024 nodes per CTA is the most the sampling scan takes: one CTA over 1 100 nodes is refused."""
    snap = _wide(1100, percentage_nodes_to_find=10, min_nodes_to_find=20)
    geo = _geometry(snap, {"VC_COMMIT_CTAS": 1}, sm_count)
    assert geo["rows"] == 5
    gpu.debug_option("VC_COMMIT_CTAS", 1)
    try:
        e = gpu.Engine(snap)
        try:
            with pytest.raises(gpu.VcError) as ei:
                e.upload()
                e.allocate()
        finally:
            e.close()
    finally:
        gpu.debug_option("VC_COMMIT_CTAS", 0)
    assert ei.value.code == abi.VC_EUNSUPPORTED
