"""The backfill kernel (k_backfill, volcano_b200/csrc/vc_backfill.cuh) on every path it takes, against the CPU oracle's
backfill() on the same session: decisions (task, node, visit, fp64 score) bit-equal, visits, fit errors and the
lastProcessedNodeIndex the action leaves.

The kernel's shortcuts engage only at some shapes, so every case asserts, worked out in Python, the precondition that
puts it on its path:
  * the instance: k_backfill<true, true> under feasible-node sampling, <true> with a live TaintToleration batch score
    (two passes per task), <false> otherwise;
  * the launch geometry (a mirror of choose_geometry): CTAs, nodes per CTA, block and sweep rows;
  * the run structure: same-group runs and consecutive placements on one node, from the oracle's pick order and decisions;
  * the tracked path of the plain instance: with VC_PROF, prof_cycles[1] counts the full sweep steps of the grid and
    prof_cycles[3] the steps CTA 0 republishes alone, both exactly as the Python mirror of the single-publisher rule
    counts them (full on a group switch and after 24 publications)."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SYNC_EVERY = 24   # publications between two all-gathers of the plain instance
SPEC_DEPTH = 32   # run-ahead entries on integer-valued sessions
HAS_TOPO = 1 << 30  # the group-key bit of pods of soft-mode topology jobs


@pytest.fixture(scope="module")
def gpu():
    from volcano_b200 import engine
    engine.init(0)
    return engine


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cfg(base, **changes):
    from volcano_b200.synth import CONFIGS
    return dataclasses.replace(CONFIGS[base], name=f"{base}-bf", **changes)


def _make(cfg):
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg)
    snap.synth_cfg = cfg
    return snap


# ---- restatements of the library's choices (preconditions only) ------------------------------------------------
def _to_find(snap):
    """d.to_find: numNodesToFind (util/scheduler_helper.go:54-73), 0 = no sampling."""
    c, N = snap.conf, snap.N
    if N <= c.min_nodes_to_find or c.percentage_nodes_to_find >= 100:
        return 0
    pct = c.percentage_nodes_to_find
    if pct <= 0:
        pct = max(50 - N // 125, c.min_percentage_nodes_to_find)
    tf = max(N * pct // 100, c.min_nodes_to_find)
    return tf if tf < N else 0


def _nta_plugin(snap):
    return "network-topology-aware" in snap.synth_cfg.plugins


def _soft_active(snap):
    return "nodeorder" in snap.synth_cfg.plugins and snap.conf.w_taint_toleration != 0 and bool(snap.n_taint_soft.any())


def _instance(snap):
    return "samp" if _to_find(snap) > 0 else "soft" if _soft_active(snap) else "plain"


def _geometry(snap, opts, sm):
    """choose_geometry on one GPU over the full node axis (every synthetic job has one role: the error cache is a no-op)."""
    assert not snap.synth_cfg.mixed_roles
    N = snap.N
    ctas = opts.get("VC_COMMIT_CTAS", 0) or sm
    block = 128
    if opts.get("VC_COMMIT_THREADS", 0):
        block = max(128, min(256, opts["VC_COMMIT_THREADS"] // 32 * 32))
    ctas = max(1, min(ctas, (N + 31) // 32))
    npc = max(32, (-(-N // ctas) + 31) // 32 * 32)
    topo_any = _nta_plugin(snap) and snap.hn_job_soft is not None and bool(snap.hn_job_soft.any())
    nta_on = _nta_plugin(snap) and snap.conf.nta_normal_pod_enable != 0
    samp_ok = _to_find(snap) == 0 or not _soft_active(snap)
    fast = not topo_any and not nta_on and samp_ok and snap.R <= 8
    if fast and not opts.get("VC_COMMIT_CTAS", 0) and npc < 128 and N >= 64 * 128:
        npc = 128
    ctas = max(1, -(-N // npc))
    if npc > block:
        block = min(256, (npc + 31) // 32 * 32)
    return {"ctas": ctas, "npc": npc, "block": block, "rows": -(-npc // block)}


def _integral(*arrays):
    return all(np.array_equal(a, np.trunc(a)) and (np.abs(a) < 9.0e15).all() for a in arrays if a.size)


def _rows_integral(snap):
    """vch::runs_exact over the node rows, the pending tasks' and the BestEffort tasks' requests (spec_depth 32 vs 1)."""
    if not _integral(snap.n_idle, snap.n_used, snap.n_releasing, snap.n_pipelined, snap.n_k8s_requested,
                     snap.n_k8s_nonzero_requested, snap.t_resreq, snap.t_k8s_req, snap.t_k8s_nonzero_req, snap.b_resreq,
                     snap.b_k8s_req, snap.b_k8s_nonzero_req):
        return False
    for rows, reqs in (((snap.n_idle, snap.n_used), (snap.t_resreq, snap.b_resreq)),
                       ((snap.n_k8s_requested,), (snap.t_k8s_req, snap.b_k8s_req)),
                       ((snap.n_k8s_nonzero_requested[:2],), (snap.t_k8s_nonzero_req[:2], snap.b_k8s_nonzero_req[:2]))):
        mrow = np.max([np.abs(r).max(axis=1) for r in rows], axis=0)
        mreq = np.max([np.abs(q).max(axis=1) if q.shape[1] else np.zeros(q.shape[0]) for q in reqs], axis=0)
        if not (mrow + 32.0 * mreq < 9.0e15).all():
            return False
    return True


def _groups(snap):
    """(class, has-bits, request rows) group of every BestEffort task, the key of the kernel's verdict cache."""
    has = snap.b_req_has.astype(np.int64)
    if _nta_plugin(snap) and snap.hn_job_soft is not None:
        has = has | (snap.hn_job_soft[snap.b_job].astype(np.int64) * HAS_TOPO)

    def cols(a):
        return np.ascontiguousarray(np.asarray(a, np.float64).T).view(np.int64)

    key = np.concatenate([snap.b_klass.astype(np.int64)[:, None], has[:, None], cols(snap.b_resreq), cols(snap.b_k8s_req),
                          cols(snap.b_k8s_nonzero_req[:2])], axis=1)
    return np.unique(key, axis=0, return_inverse=True)[1].ravel()


def _steps(snap, order, ref):
    """(group, node or -1) per pick position, from the oracle's decisions."""
    dec, _, fe = ref
    node = np.full(snap.B, -1, np.int64)
    node[dec["task"]] = dec["node"]
    assert len(dec) + len(fe) == len(order)
    return _groups(snap)[order], node[order]


def _runs(groups, nodes):
    """[(group, node, length)]: maximal runs of consecutive pick positions of one group placed on one node."""
    out = []
    for g, n in zip(groups, nodes):
        if out and n >= 0 and out[-1][0] == g and out[-1][1] == n:
            out[-1][2] += 1
        else:
            out.append([g, n, 1])
    return [tuple(r) for r in out if r[1] >= 0]


def _tracked(groups, nodes, npc):
    """The single-publisher rule of k_backfill<false>: a step is a full all-gather when its group differs from the
    previous task's, or after 24 publications since the last one; otherwise only the previous owner (the CTA of the
    previous placement, none after a task without a node) sweeps and publishes."""
    tb_group, prev_owner, since = -1, -1, 0
    full = resync = rep0 = silent = 0
    for g, n in zip(groups, nodes):
        if tb_group != g or since >= SYNC_EVERY:
            full += 1
            resync += tb_group == g
            since = 0
        else:
            rep0 += prev_owner == 0
            silent += prev_owner < 0
            if prev_owner >= 0:
                since += 1
        tb_group = g
        prev_owner = n // npc if n >= 0 else -1
    return {"full": full, "resync": resync, "republish0": rep0, "silent": silent}


def _passes(snap, nodes):
    """Full sweep passes of the untracked instances: one per task, two for a placed task when the batch score is live."""
    two = _soft_active(snap)
    return len(nodes) + (int((nodes >= 0).sum()) if two else 0)


# ---- running both sides --------------------------------------------------------------------------------------------
def _oracle(snap, alloc=True, threads=4):
    from oracle import pyoracle
    from oracle.pyoracle import OracleSession
    o = OracleSession(snap, threads=threads)
    a = o.allocate() if alloc else None
    a_last = int(pyoracle.lib().vco_last_processed_node_index(o.h))
    order = o.backfill_pick_order()
    b = o.backfill()
    last = int(pyoracle.lib().vco_last_processed_node_index(o.h))
    o.close()
    return {"alloc": a, "alloc_last": a_last, "order": order, "bf": b, "last": last}


def _library(gpu, snap, opts=None, alloc=True):
    opts = dict(opts or {})
    for k, v in opts.items():
        gpu.debug_option(k, v)
    try:
        e = gpu.Engine(snap)
        e.upload()
        a = e.allocate() if alloc else None
        gpu.debug_option("VC_PROF", 1)
        b = e.backfill()
        gpu.debug_option("VC_PROF", 0)
        e.close()
    finally:
        for k in list(opts) + ["VC_PROF"]:
            gpu.debug_option(k, 0)
    return a, b


def _same(got, ref, what):
    dec, vis, fe = ref
    assert np.array_equal(got.visits, vis), f"{what}: visits differ"
    for f in ("task", "node", "kind", "visit"):
        bad = np.flatnonzero(got.decisions[f] != dec[f]) if len(got.decisions) == len(dec) else [-1]
        assert len(got.decisions) == len(dec) and not len(bad), f"{what}: decision {f} differs from index {bad[0]}"
    assert np.array_equal(got.decisions["score"].view(np.int64), dec["score"].view(np.int64)), f"{what}: fp64 scores differ"
    assert np.array_equal(got.fit_errors, fe), f"{what}: fit errors differ"


def _check(snap, got, ref, alloc=True):
    a, b = got
    if alloc:
        _same(a, ref["alloc"], "allocate")
        assert a.stats["last_processed_node_index"] == ref["alloc_last"]
    _same(b, ref["bf"], "backfill")
    assert b.stats["last_processed_node_index"] == ref["last"]


def _check_path(snap, b, ref, geo):
    """prof_cycles[1] / [3] against the mirror of the instance the session takes; returns the mirror's counts."""
    groups, nodes = _steps(snap, ref["order"], ref["bf"])
    prof = b.stats["prof_cycles"]
    if _instance(snap) == "plain":
        t = _tracked(groups, nodes, geo["npc"])
        assert prof[1] == t["full"], (prof[1], t)
        assert prof[3] == t["republish0"], (prof[3], t)
        return t
    assert prof[1] == _passes(snap, nodes) and prof[3] == 0, (prof[1], prof[3], _passes(snap, nodes))
    return None


# ---- sessions of long same-group runs -------------------------------------------------------------------------------
# Backfill's node order is nodeorder's mostrequested alone: the node that took a pod scores at least as high as before,
# so it keeps winning until its pod cap ends the run. The run nodes have cpu and memory fully requested (score 100, the
# top: ties go to the lowest index, so the runs come in node order; no room for a regular pod, so allocate leaves their
# pod slots alone) and `length` free pod slots. Y is the one node labelled with bit 63, which class `cls_y` selects.
RUN_NODES = (3, 5, 40, 100, 300, 420, 650)
RUN_LENGTHS = (33, 1, 64, 31, 65, 30, 32)
NODE_Y = 690
LABEL_Y = np.uint64(1) << np.uint64(63)
INTERLEAVE = (5, 10)  # run index, offset: one task of Y's class in the middle of that run (A A B A A)


def _reserve(snap, n, free):
    from volcano_b200.synth import D_CPU, D_MEM, D_PODS
    for d, k in ((D_CPU, 0), (D_MEM, 1)):
        a = snap.n_allocatable[d, n]
        snap.n_used[d, n], snap.n_idle[d, n] = a, 0.0
        snap.n_k8s_requested[k, n] = snap.n_k8s_nonzero_requested[k, n] = a
    snap.n_taint_hard[:, n] = 0
    snap.n_pod_count[n] = snap.n_max_tasks[n] - free
    snap.n_used[D_PODS, n] = snap.n_pod_count[n]
    snap.n_idle[D_PODS, n] = free


def _packed(head=0, y_free=1, interleave=True, extra=60):
    """One job holds every BestEffort pod. Pick positions [0, head) and, with `interleave`, one position inside run
    INTERLEAVE take class `cls_y` (Y only); the rest take class 0 (no selector, no toleration)."""
    from oracle.pyoracle import OracleSession
    B = head + sum(RUN_LENGTHS) + (1 if interleave else 0) + extra
    snap = _make(_cfg("small_bf", plugins="priority+gang+drf+predicates+proportion+nodeorder", n_besteffort=B,
                      besteffort_jobs=1))
    c = snap.conf
    c.w_most, c.w_least, c.w_balanced, c.w_node_affinity, c.w_taint_toleration = 1, 0, 0, 0, 0
    for n, free in zip(RUN_NODES, RUN_LENGTHS):
        _reserve(snap, n, free)
    _reserve(snap, NODE_Y, y_free)
    snap.n_label_bits[0] &= ~LABEL_Y
    snap.n_label_bits[0, NODE_Y] |= LABEL_Y
    use = np.bincount(snap.t_klass, minlength=snap.C)
    cls_y = 1 + int(np.argmin(use[1:]))  # the class fewest regular pods use
    snap.c_selector[cls_y] = 0
    snap.c_selector[cls_y, 0] = LABEL_Y
    o = OracleSession(snap, threads=4)
    o.allocate()
    order = o.backfill_pick_order()
    o.close()
    assert len(order) == B
    klass = np.zeros(B, np.int32)
    klass[:head] = cls_y
    if interleave:
        r, off = INTERLEAVE
        klass[head + sum(RUN_LENGTHS[:r]) + off] = cls_y
    snap.b_klass[order] = klass
    snap.cls_y = cls_y
    return snap


def _nonintegral():
    snap = _packed()
    snap.n_k8s_nonzero_requested[0, 1::7] += 0.1  # k8s non-zero requested sums of x.1 on every 7th node
    return snap


SESSIONS = {
    "runs": lambda: _packed(),
    "single_node": lambda: _packed(head=50, y_free=20, interleave=False),
    "runs_nonintegral": _nonintegral,
}
_cache = {}


def _session(name):
    """name -> (snapshot, oracle result); the oracle runs once per session."""
    if name not in _cache:
        snap = SESSIONS[name]()
        _cache[name] = (snap, _oracle(snap))
    return _cache[name]


def _assert_runs(snap, ref, geo):
    groups, nodes = _steps(snap, ref["order"], ref["bf"])
    runs = _runs(groups, nodes)
    by_node = {}
    for g, n, length in runs:
        by_node.setdefault(n, []).append(length)
    # the run nodes fill in node order, each to its pod cap, and the regular nodes take the rest
    for i, (n, free) in enumerate(zip(RUN_NODES, RUN_LENGTHS)):
        want = [INTERLEAVE[1], free - INTERLEAVE[1]] if i == INTERLEAVE[0] else [free]
        assert by_node.get(n) == want, (n, by_node.get(n), want)
    lengths = [r[2] for r in runs]
    assert {1, 31, 32, 33, 64, 65} <= set(lengths), lengths
    assert max(lengths) >= 65
    return groups, nodes, runs


# ---- 1. long runs on the plain instance; 3. depth 1 -------------------------------------------------------------
@pytest.mark.parametrize("depth1", [0, 1], ids=["spec32", "depth1"])
def test_long_runs(depth1, gpu, sm_count):
    """Runs of 1 to 65 pods on one node: 32 run-ahead entries exhausted and recomputed (33, 64, 65), runs ended by the
    pod cap partway through a computed run-ahead (1, 31, 33, 65), resyncs after 24 publications, CTA 0 republishing,
    and A A B A A where the run-ahead of A stays pending while B lands in another CTA. VC_BACKFILL_DEPTH1 gives the same
    result through the depth-1 path."""
    snap, ref = _session("runs")
    geo = _geometry(snap, {}, sm_count)
    assert _instance(snap) == "plain" and _rows_integral(snap)
    assert geo == {"ctas": 22, "npc": 32, "block": 128, "rows": 1}
    groups, nodes, runs = _assert_runs(snap, ref, geo)
    t = _tracked(groups, nodes, geo["npc"])
    assert t["resync"] >= 5 and t["republish0"] >= 30, t
    # A A B A A: B is Y's only pod, placed alone (score 0.0) in another CTA than the A run around it
    r, off = INTERLEAVE
    pos = sum(RUN_LENGTHS[:r]) + off
    assert groups[pos] != groups[pos - 1] == groups[pos + 1] and nodes[pos] == NODE_Y
    assert nodes[pos - 1] == nodes[pos + 1] == RUN_NODES[r] and NODE_Y // geo["npc"] != RUN_NODES[r] // geo["npc"]
    y = ref["bf"][0][ref["bf"][0]["node"] == NODE_Y]
    assert len(y) == 1 and y["score"][0] == 0.0
    # on the regular nodes after the run nodes a node's score moves within a run (the run-ahead's row view matters)
    tail = ref["bf"][0][sum(RUN_LENGTHS) + 1:]
    assert ((tail["node"][1:] == tail["node"][:-1]) & (tail["score"][1:] != tail["score"][:-1])).any()
    _, b = got = _library(gpu, snap, {"VC_BACKFILL_DEPTH1": depth1})
    _check(snap, got, ref)
    _check_path(snap, b, ref, geo)


def test_single_feasible_node_then_none(gpu, sm_count):
    """A group with one feasible node: every placement takes the one-candidate shortcut (score 0.0) up to the node's pod
    cap, then the group's tasks find no node (steps without a previous owner in the middle of a tracked run), then a
    group switch."""
    snap, ref = _session("single_node")
    geo = _geometry(snap, {}, sm_count)
    assert _instance(snap) == "plain"
    groups, nodes = _steps(snap, ref["order"], ref["bf"])
    assert (groups[:50] == groups[0]).all() and groups[50] != groups[0]
    assert (nodes[:20] == NODE_Y).all() and (nodes[20:50] == -1).all() and nodes[50] >= 0
    dec = ref["bf"][0]
    assert (dec["score"][dec["node"] == NODE_Y] == 0.0).all() and len(ref["bf"][2]) == 30
    t = _tracked(groups, nodes, geo["npc"])
    assert t["silent"] == 29, t  # no CTA sweeps on the failing steps after the first
    got = _library(gpu, snap)
    _check(snap, got, ref)
    _check_path(snap, got[1], ref, geo)


@pytest.mark.parametrize("depth1", [0, 1], ids=["auto", "depth1"])
def test_nonintegral_rows_take_depth1(depth1, gpu, sm_count):
    """Rows that are not integer-valued (non-zero requested sums of x.1): the run-ahead covers one pod by itself."""
    snap, ref = _session("runs_nonintegral")
    assert not _rows_integral(snap) and _instance(snap) == "plain"
    geo = _geometry(snap, {}, sm_count)
    _assert_runs(snap, ref, geo)
    got = _library(gpu, snap, {"VC_BACKFILL_DEPTH1": depth1})
    _check(snap, got, ref)
    _check_path(snap, got[1], ref, geo)


# ---- 4. geometry -----------------------------------------------------------------------------------------------------
GEOMETRY = [
    # N, tasks, BestEffort pods, options, expected geometry, backfill alone
    (1, 40, 30, {}, {"ctas": 1, "npc": 32, "block": 128, "rows": 1}, False),
    (31, 200, 200, {}, {"ctas": 1, "npc": 32, "block": 128, "rows": 1}, False),
    (33, 200, 200, {}, {"ctas": 2, "npc": 32, "block": 128, "rows": 1}, False),
    (700, 4000, 3000, {}, {"ctas": 22, "npc": 32, "block": 128, "rows": 1}, False),
    (8191, 2000, 1500, {}, {"ctas": 128, "npc": 64, "block": 128, "rows": 1}, False),
    (8192, 2000, 1500, {}, {"ctas": 64, "npc": 128, "block": 128, "rows": 1}, False),
    (10_001, 2000, 1500, {}, {"ctas": 79, "npc": 128, "block": 128, "rows": 1}, False),
    (40_000, 1000, 400, {}, {"ctas": 125, "npc": 320, "block": 256, "rows": 2}, False),
    # few CTAs: blocks of 128 and 256 threads while a CTA's nodes fit one block, several sweep rows beyond (a block
    # is 256 threads from 256 nodes per CTA on). The commit kernel keeps more per node in shared memory than backfill
    # and cannot hold 672 or 800 nodes per CTA: those sessions run backfill alone.
    (300, 1500, 1000, {"VC_COMMIT_CTAS": 3}, {"ctas": 3, "npc": 128, "block": 128, "rows": 1}, False),
    (300, 1500, 1000, {"VC_COMMIT_CTAS": 3, "VC_COMMIT_THREADS": 256}, {"ctas": 3, "npc": 128, "block": 256, "rows": 1}, False),
    (2000, 2000, 2000, {"VC_COMMIT_CTAS": 3}, {"ctas": 3, "npc": 672, "block": 256, "rows": 3}, True),
    (800, 1000, 1500, {"VC_COMMIT_CTAS": 1, "VC_COMMIT_THREADS": 256}, {"ctas": 1, "npc": 800, "block": 256, "rows": 4}, True),
]


@pytest.mark.parametrize("N,T,B,opts,want,alone", GEOMETRY,
                         ids=[f"n{g[0]}-" + "-".join(f"{k[10:].lower()}{v}" for k, v in g[3].items()) for g in GEOMETRY])
def test_geometry(N, T, B, opts, want, alone, gpu, sm_count):
    snap = _make(_cfg("cfg2_bf", n_nodes=N, n_tasks=T, n_besteffort=B))
    if N < 64:  # no hard taint on a handful of nodes, so that pods land
        snap.n_taint_hard[:] = 0
    geo = _geometry(snap, opts, sm_count)
    assert geo == want and _instance(snap) == "plain"
    ref = _oracle(snap, alloc=not alone)
    assert len(ref["bf"][0]) > 0
    got = _library(gpu, snap, opts, alloc=not alone)
    _check(snap, got, ref, alloc=not alone)
    t = _check_path(snap, got[1], ref, geo)
    assert t["full"] < len(ref["order"])  # some steps republish alone


# ---- 5. sampling -----------------------------------------------------------------------------------------------------
SAMPLING = [
    # name, base, (pct, min nodes, start), options, backfill alone (the start is the configured index, not allocate's)
    ("window_in_one_cta", "small_bf", (1, 5, 3), {}, True),
    ("window_over_ctas", "small_bf", (15, 20, 40), {}, True),
    ("wrap_from_last_cta", "small_bf", (5, 30, 690), {}, True),
    ("fewer_feasible", "small_bf", (20, 10, 100), {}, False),
    ("carried_from_allocate", "small_bf", (10, 20, 0), {}, False),
    ("adaptive", "small_bf", (0, 100, 0), {}, False),
    ("alone_start_past_n", "small_bf", (10, 20, 700 + 123), {}, True),
    ("four_rows", "small_bf", (10, 20, 1500), {"VC_COMMIT_CTAS": 2}, True),
    ("soft_window_over_ctas", "small_soft_bf", (25, 10, 17), {}, True),
    ("soft_wrap_from_last_cta", "small_soft_bf", (5, 30, 290), {}, True),
    ("soft_fewer_feasible", "small_soft_bf", (30, 10, 0), {}, False),
    ("soft_carried_from_allocate", "small_soft_bf", (10, 20, 5), {}, False),
    ("soft_alone_start_past_n", "small_soft_bf", (10, 20, 300 + 299), {}, True),
    ("soft_four_rows", "small_soft_bf", (10, 20, 1500), {"VC_COMMIT_CTAS": 2}, True),
]


def _samp_snapshot(name, base, args):
    pct, mn, start = args
    kw = {"n_nodes": 1600, "n_tasks": 3000, "n_besteffort": 1500} if "four_rows" in name else {}
    snap = _make(_cfg(base, **kw))
    if "fewer_feasible" in name:  # every BestEffort pod in one class that selects one zone (~1/16 of the nodes)
        zone = snap.C - 1
        snap.c_selector[zone] = 0
        snap.c_selector[zone, 0] = np.uint64(1) << np.uint64(5)
        snap.b_klass[:] = zone
    snap.conf.percentage_nodes_to_find, snap.conf.min_nodes_to_find, snap.conf.last_processed_node_index = pct, mn, start
    return snap


@pytest.mark.parametrize("name,base,args,opts,alone", SAMPLING, ids=[s[0] for s in SAMPLING])
def test_sampling(name, base, args, opts, alone, gpu, sm_count):
    snap = _samp_snapshot(name, base, args)
    geo = _geometry(snap, opts, sm_count)
    tf, N = _to_find(snap), snap.N
    start = args[2] % N
    assert _instance(snap) == "samp" and tf > 0
    assert _soft_active(snap) == name.startswith("soft")
    ref = _oracle(snap, alloc=not alone, threads=1)
    first = start if alone else ref["alloc_last"]  # where backfill's scan starts
    ok = _static_ok(snap, ref["order"][0])
    processed = _scan(ok, first, tf)  # nodes the first task's scan looks at (every node is below its pod cap at open)
    lo, hi = first // geo["npc"], (first + processed - 1) % N // geo["npc"]
    if "window_in_one_cta" in name:
        assert alone and processed < N and lo == hi and first % geo["npc"] > 0
    if "window_over_ctas" in name:
        assert alone and hi - lo >= 2
    if "wrap" in name:
        assert alone and lo == geo["ctas"] - 1 and first + processed > N
    if "fewer_feasible" in name:  # no task finds to_find nodes: every scan covers all N nodes and the index returns
        assert ok.sum() < tf and ref["last"] == first
    if alone:
        assert (snap.n_pod_count < snap.n_max_tasks).all()
    if "past_n" in name:
        assert alone and args[2] >= N
    if not alone:  # the start index comes from allocate under sampling
        assert first != start
    if "four_rows" in name:
        assert geo["rows"] == 4 and geo["npc"] == 800
    assert len(ref["bf"][0]) > 0
    got = _library(gpu, snap, opts, alloc=not alone)
    _check(snap, got, ref, alloc=not alone)
    _check_path(snap, got[1], ref, geo)


def _static_ok(snap, t):
    """The predicates of BestEffort task t on every node at open: nodeSelector and hard taints."""
    c = snap.b_klass[t]
    sel = snap.c_selector[c, 0]
    ok = (snap.n_label_bits[0] & sel) == sel
    return ok & ((snap.n_taint_hard[0] & ~snap.c_tolerated_hard[c, 0]) == 0)


def _scan(ok, start, tf):
    """processedNodes of the single-worker scan: nodes looked at until `tf` feasible ones are found (N when fewer)."""
    N = len(ok)
    hits = np.flatnonzero(np.roll(ok, -start))
    return int(hits[tf - 1]) + 1 if len(hits) >= tf else N


@pytest.mark.parametrize("base", ["small_bf", "small_soft_bf"])
def test_sampling_refuses_more_than_four_rows(base, gpu, sm_count):
    """1 024 nodes per CTA is the most the sampling scan takes (4 rows of 256 threads): one CTA over 2 000 nodes is refused."""
    big = _make(_cfg(base, n_nodes=2000, n_tasks=2000, n_besteffort=500))
    big.conf.percentage_nodes_to_find, big.conf.min_nodes_to_find = 10, 20
    geo = _geometry(big, {"VC_COMMIT_CTAS": 1}, sm_count)
    assert geo["npc"] > 1024 and geo["rows"] > 4
    gpu.debug_option("VC_COMMIT_CTAS", 1)
    try:
        e = gpu.Engine(big)
        with pytest.raises(gpu.VcError) as ei:
            e.upload()
            e.allocate()
            e.backfill()
        e.close()
    finally:
        gpu.debug_option("VC_COMMIT_CTAS", 0)
    from volcano_b200 import abi
    assert ei.value.code == abi.VC_EUNSUPPORTED


def test_sampling_finds_no_node_is_refused(gpu):
    """min_nodes_to_find 0 and 10 nodes at 5 %: numNodesToFind is 0. The reference finds no node (and moves its index by
    an amount its workers decide); allocate and backfill refuse the session instead of scheduling over every node."""
    from volcano_b200 import abi
    snap = _make(_cfg("tiny_bf", n_nodes=10, n_tasks=40, n_besteffort=20))
    snap.conf.percentage_nodes_to_find, snap.conf.min_nodes_to_find = 5, 0
    assert snap.N * 5 // 100 == 0
    ref = _oracle(snap)
    assert len(ref["alloc"][0]) == 0 and len(ref["bf"][0]) == 0 and len(ref["bf"][2]) == len(ref["order"]) > 0
    e = gpu.Engine(snap)
    e.upload()
    with pytest.raises(gpu.VcError) as ei:
        e.allocate()
    assert ei.value.code == abi.VC_EUNSUPPORTED
    with pytest.raises(gpu.VcError) as ei:
        e.backfill()
    assert ei.value.code == abi.VC_EUNSUPPORTED
    e.close()


def test_launch_refused_for_shared_memory_leaves_no_error(gpu):
    """800 nodes per CTA do not fit the commit kernel's shared memory: allocate reports the CUDA error, and the next
    session on a new engine runs as if nothing had happened (the error is not left for its checks to find)."""
    from volcano_b200 import abi
    snap = _make(_cfg("cfg2_bf", n_nodes=800, n_tasks=1000, n_besteffort=1500))
    gpu.debug_option("VC_COMMIT_CTAS", 1)
    try:
        e = gpu.Engine(snap)
        e.upload()
        with pytest.raises(gpu.VcError) as ei:
            e.allocate()
        e.close()
    finally:
        gpu.debug_option("VC_COMMIT_CTAS", 0)
    assert ei.value.code == abi.VC_ECUDA
    ref = _oracle(snap)
    _check(snap, _library(gpu, snap), ref)


# ---- 6. the two-pass SOFT instance at more CTAs ---------------------------------------------------------------------
SOFT = [
    ("n2000", {"n_nodes": 2000, "n_tasks": 3000, "n_besteffort": 1500}, None),
    ("n2000_adaptive", {"n_nodes": 2000, "n_tasks": 3000, "n_besteffort": 1500}, 0),
    ("n10000", {"n_tasks": 3000, "n_besteffort": 1500}, None),
    ("n10000_adaptive", {"n_tasks": 3000, "n_besteffort": 1500}, 0),
]


@pytest.mark.parametrize("name,kw,pct", SOFT, ids=[s[0] for s in SOFT])
def test_soft_two_pass(name, kw, pct, gpu, sm_count):
    snap = _make(_cfg("cfg2_soft", **kw))
    if pct is not None:
        snap.conf.percentage_nodes_to_find = pct
    geo = _geometry(snap, {}, sm_count)
    assert _soft_active(snap) and _instance(snap) == ("soft" if pct is None else "samp")
    assert geo["ctas"] >= 60
    ref = _oracle(snap, threads=4 if pct is None else 1)
    dec = ref["bf"][0]
    assert len(dec) > 0 and (dec["score"] != 0.0).any()
    got = _library(gpu, snap)
    _check(snap, got, ref)
    _check_path(snap, got[1], ref, geo)


def test_soft_topology_jobs_with_besteffort_pods(gpu, sm_count):
    """network-topology-aware with soft-mode topology jobs that carry BestEffort pods next to normal pods: the static
    hypernode-binpack entry applies to the normal pods only (the topology flag splits the groups)."""
    snap = _make(_cfg("small_topo_bf", n_nodes=2000, n_tasks=4000, n_besteffort=2500))
    soft_be = snap.hn_job_soft[snap.b_job].astype(bool)
    assert soft_be.any() and (~soft_be).any() and _nta_plugin(snap)
    geo = _geometry(snap, {}, sm_count)
    ref = _oracle(snap)
    groups, nodes = _steps(snap, ref["order"], ref["bf"])
    assert ((nodes >= 0) & soft_be[ref["order"]]).any() and ((nodes >= 0) & ~soft_be[ref["order"]]).any()
    got = _library(gpu, snap)
    _check(snap, got, ref)
    _check_path(snap, got[1], ref, geo)


# ---- 7. repeated cycles on one engine -----------------------------------------------------------------------------
def test_repeated_cycles_on_one_engine(gpu):
    """allocate -> backfill three times on one upload, then an upload with more BestEffort pods (the device slab grows):
    every run equals the oracle, and backfill without a new allocate is refused."""
    small = _make(_cfg("small_bf", n_besteffort=600))
    big = _make(_cfg("small_bf", n_besteffort=3000))
    assert np.array_equal(small.t_resreq, big.t_resreq) and big.B > small.B
    ref_s, ref_b = _oracle(small), _oracle(big)
    e = gpu.Engine(small)
    try:
        e.upload()
        for _ in range(3):
            _check(small, (e.allocate(), e.backfill()), ref_s)
        e.upload(big)
        _check(big, (e.allocate(), e.backfill()), ref_b)
        with pytest.raises(gpu.VcError):
            e.backfill()
    finally:
        e.close()


# ---- 8. full size --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pct", [None, 0], ids=["default", "adaptive_sampling"])
def test_cfg2_bf_full_size(pct, gpu, sm_count):
    """cfg2_bf (10 000 nodes, 100 000 pods, 20 000 BestEffort pods) at the default settings and under the reference's
    adaptive sampling (percentage-nodes-to-find 0: 5 % of the nodes)."""
    import os
    snap = _make(_cfg("cfg2_bf"))
    if pct is not None:
        snap.conf.percentage_nodes_to_find = pct
    geo = _geometry(snap, {}, sm_count)
    assert _instance(snap) == ("plain" if pct is None else "samp")
    ref = _oracle(snap, threads=max(1, min(16, os.cpu_count() or 1)) if pct is None else 1)
    assert len(ref["bf"][0]) > 10_000
    got = _library(gpu, snap)
    _check(snap, got, ref)
    _check_path(snap, got[1], ref, geo)
