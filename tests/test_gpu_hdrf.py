"""Hierarchical drf (drf's enableHierarchy) on the H100: both commit kernels against the hdrf oracle (tools/hdrf_oracle:
the tree recomputed in full before every queue-heap operation). Decisions, visits, fit errors and fp64 scores identical."""
import numpy as np
import pytest

from tests import hdrf_common as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    from volcano_b200 import engine
    engine.init(0)
    return engine


def _same(res, dec, vis, fe):
    assert np.array_equal(res.visits["job"], vis["job"])
    assert np.array_equal(res.visits["outcome"], vis["outcome"])
    assert np.array_equal(res.visits["n_ops"], vis["n_ops"])
    assert np.array_equal(res.visits["first_op"], vis["first_op"])
    for f in ("task", "node", "kind", "visit"):
        assert np.array_equal(res.decisions[f], dec[f]), f
    assert np.array_equal(res.decisions["score"], dec["score"])
    assert np.array_equal(np.sort(res.fit_errors), np.sort(fe))


def _run(gpu, snap, generic=False):
    gpu.debug_option("VC_COMMIT_GENERIC", 1 if generic else 0)
    try:
        res = gpu.gpu_engine(snap)
    finally:
        gpu.debug_option("VC_COMMIT_GENERIC", 0)
    assert res.stats["commit_kernel"] == (0 if generic else 1), res.stats
    return res


@pytest.mark.parametrize("generic", [False, True], ids=["fast", "generic"])
@pytest.mark.parametrize("make", [H.rescaling_case, H.blocking_case], ids=["rescaling", "blocking"])
def test_upstream_cases(gpu, make, generic):
    case = make()
    snap = case.RegisterSession(H.tiers())
    res = _run(gpu, snap, generic)
    dec, vis, fe = H.oracle_for(snap, case.Queues).allocate()
    _same(res, dec, vis, fe)


def _session(cfg, seed, sampling=False, swap=False):
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg, seed)
    rng = np.random.default_rng(1000 + seed)
    hier, wts = H.random_tree(snap, rng)
    if sampling:
        snap.conf.percentage_nodes_to_find = 0
    if swap:
        H.swap_queue_order(snap)
    return snap, hier, wts


# (config, seeds): tiny / small on the plain instance, tiny_fut (FUT), small_fut_soft (FUT + SOFT); 120 sessions in all.
# Feasible-node sampling takes effect only above min-nodes-to-find (100 nodes): it is switched on for every other 700-node
# "small" session, where the adaptive percentage gives 315 candidates per task (the SAMP instance of k_commit_fast).
FAMILY = [("tiny", range(0, 40)), ("small", range(0, 16)), ("tiny_fut", range(0, 24)), ("small_fut_soft", range(0, 16)),
          ("tiny", range(40, 64))]


def _to_find(snap):
    c = snap.conf
    n, pct = snap.N, c.percentage_nodes_to_find
    if n <= c.min_nodes_to_find or pct >= 100:
        return n
    adaptive = pct if pct > 0 else max(50 - n // 125, c.min_percentage_nodes_to_find)
    return max(n * adaptive // 100, c.min_nodes_to_find)


@pytest.mark.parametrize("cfg,seeds", FAMILY, ids=[f"{c}-{s.start}" for c, s in FAMILY])
def test_random_trees_vs_oracle(gpu, cfg, seeds):
    """Random trees (up to 4 levels, shared nodes, root-level queues, clamped weights), both tier orders of drf and
    proportion, with and without feasible-node sampling, on the incremental kernel and the general one."""
    n = 0
    for seed in seeds:
        sampling = cfg == "small" and seed % 2 == 1
        swap = seed % 2 == 1 if cfg != "small" else seed % 4 >= 2
        snap, hier, wts = _session(cfg, seed, sampling, swap)
        assert (_to_find(snap) < snap.N) == sampling  # sampling is in force exactly where it is asked for
        dec, vis, fe = H.HdrfOracle(snap, hier, wts).allocate()
        generic = seed % 4 == 3
        res = _run(gpu, snap, generic)
        _same(res, dec, vis, fe)
        n += 1
    assert n == len(seeds)


def test_heap_case_on_device(gpu):
    """The rescaling case is one where an arg-min over live keys serves queues in another order than the Go heap; the
    device follows the heap."""
    case = H.rescaling_case()
    snap = case.RegisterSession(H.tiers())
    argmin = H.oracle_for(snap, case.Queues).allocate(argmin=True)[0]
    res = _run(gpu, snap)
    assert not np.array_equal(res.decisions["task"], argmin["task"])


def test_preempt_reclaim_refused(gpu):
    """vc_preempt_run / vc_reclaim_run refuse hdrf sessions (VC_EUNSUPPORTED) and leave the session as it was: an allocate
    run afterwards still matches the oracle."""
    from volcano_b200.engine import Engine, VcError
    case = H.rescaling_case()
    snap = case.RegisterSession(H.tiers())
    e = Engine(snap)
    e.upload()
    for act in (e.preempt, e.reclaim):
        with pytest.raises(VcError) as ei:
            act()
        assert ei.value.code == -4  # VC_EUNSUPPORTED
    res = e.allocate()
    dec, vis, fe = H.oracle_for(snap, case.Queues).allocate()
    _same(res, dec, vis, fe)
    e.close()


def test_dense_pass_unchanged(gpu):
    """The dense mask + score pass does not read queue order: identical matrices with and without the table."""
    from volcano_b200.engine import Engine
    snap, _, _ = _session("small", 3)
    e = Engine(snap)
    e.upload()
    a = e.score_matrix()
    snap.clear_hdrf()
    e2 = Engine(snap)
    e2.upload()
    b = e2.score_matrix()
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    e.close(); e2.close()


def test_mid_size_both_kernels(gpu):
    """cfg3's shape (16 queues, drf + proportion) at 2 000 nodes: a 4-department x 4-team tree with unequal weights."""
    from volcano_b200.synth import SynthConfig, make_snapshot
    cfg = SynthConfig("mid16", 2_000, 20_000, 16, "priority+gang+drf+predicates+proportion+nodeorder+binpack", hdrf=(4, 4))
    snap = make_snapshot(cfg, 7)
    dec, vis, fe = H.HdrfOracle(snap, *_annotations(cfg, snap.Q)).allocate()
    assert len(dec) > 1000
    for generic in (False, True):
        _same(_run(gpu, snap, generic), dec, vis, fe)


def _annotations(cfg, Q):
    depts, teams = cfg.hdrf
    return ([f"root/dept{(q // teams) % depts}/team{q % teams}" for q in range(Q)],
            [f"1/{1 + (q // teams) % depts}/{1 + 2 * (q % teams)}" for q in range(Q)])


@pytest.mark.parametrize("generic", [False, True], ids=["fast", "generic"])
def test_cfg3_hdrf_full_size(gpu, generic):
    """cfg3_hdrf at full size (10 000 nodes x 100 000 tasks, 16 queues under 4 x 4 teams) on both kernels."""
    from volcano_b200.synth import CONFIGS, make_snapshot
    import os
    snap = make_snapshot("cfg3_hdrf")
    threads = max(1, min(16, len(os.sched_getaffinity(0))))
    dec, vis, fe = H.HdrfOracle(snap, *_annotations(CONFIGS["cfg3_hdrf"], snap.Q), threads=threads).allocate()
    assert len(dec) > 90_000
    _same(_run(gpu, snap, generic), dec, vis, fe)


@pytest.mark.parametrize("cfg,seeds", [("tiny_bf", range(0, 12)), ("small_bf", range(0, 4))])
def test_allocate_then_backfill(gpu, cfg, seeds):
    """Allocate followed by backfill: pickUpPendingTasks orders queues by the hdrf chain on the tree allocate left."""
    from volcano_b200.engine import Engine
    for seed in seeds:
        snap, hier, wts = _session(cfg, seed, swap=seed % 2 == 1)
        o = H.HdrfOracle(snap, hier, wts)
        ref_a = o.allocate()
        ref_b = o.backfill()
        assert len(ref_b[0]) > 0
        e = Engine(snap)
        _same(e.allocate(), *ref_a)
        _same(e.backfill(), *ref_b)
        e.close()


def test_backfill_without_hdrf_queue_order(gpu, oracle_engine):
    """With the table set but drf's EnabledQueueOrder off, the queue order is proportion's alone: allocate and backfill
    equal the plain oracle's."""
    from volcano_b200.engine import Engine
    from oracle.pyoracle import OracleSession
    snap, hier, wts = _session("tiny_bf", 3)
    c = snap.conf
    for i in range(c.n_plugins):
        if c.plugins[i].plugin == 3:  # VC_PLUGIN_DRF
            c.plugins[i].enabled &= ~0x010  # VC_EN_QUEUE_ORDER
    o = OracleSession(snap)
    ref_a, ref_b = o.allocate(), o.backfill()
    e = Engine(snap)
    _same(e.allocate(), *ref_a)
    _same(e.backfill(), *ref_b)
    e.close()


def test_fuzz_api_hdrf_family(gpu):
    """A slice of tools/fuzz_api.py's hdrf family (API-level clusters, random trees, both tier orders, sampling, nominated
    nodes, BestEffort pods): allocate, then backfill where the action list has it, against the hdrf oracle."""
    import importlib.util
    import os
    from volcano_b200.engine import Engine
    spec = importlib.util.spec_from_file_location("fuzz_api", os.path.join(H.ROOT, "tools", "fuzz_api.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sessions = backfills = 0
    for seed in range(1, 141):
        tc, tiers, actions, hier, wts = mod.make_hdrf_case(seed)
        if not tiers:
            continue
        snap = tc.RegisterSession(tiers, actions=actions, **tc.conf_kw)
        if snap.T == 0 or snap.N == 0:
            continue
        o = H.HdrfOracle(snap, hier, wts)
        assert o.attach_rc == 0
        e = Engine(snap)
        _same(e.allocate(), *o.allocate())
        sessions += 1
        if "backfill" in actions and snap.B > 0 and mod.backfill_supported(tiers, tc.conf_kw):
            _same(e.backfill(), *o.backfill())
            backfills += 1
        e.close()
    assert sessions >= 100 and backfills >= 30
