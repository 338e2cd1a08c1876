"""GPU parity tests proper: the CUDA path, called through the C ABI (libvcalloc.so), against the CPU oracle
and the reference's golden vectors.  Placements must be identical (same node per task, same order, same
visit outcomes); fp64 scores must agree within 1e-6 (north_star) — in practice they are bit-equal because
both sides execute the same IEEE operations in the same order."""
import numpy as np
import pytest

from tests.golden import reference_cases as G

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-6


@pytest.fixture(scope="module")
def gpu():
    from volcano_b200 import engine
    engine.init(0)
    return engine


def _assert_same(a, b):
    assert len(a.visits) == len(b.visits), (len(a.visits), len(b.visits))
    assert np.array_equal(a.visits["job"], b.visits["job"])
    assert np.array_equal(a.visits["outcome"], b.visits["outcome"])
    assert np.array_equal(a.visits["n_ops"], b.visits["n_ops"])
    assert np.array_equal(a.visits["first_op"], b.visits["first_op"])
    assert len(a.decisions) == len(b.decisions)
    for f in ("task", "node", "kind", "visit"):
        assert np.array_equal(a.decisions[f], b.decisions[f]), f
    assert np.allclose(a.decisions["score"], b.decisions["score"], rtol=0, atol=SCORE_TOL)
    assert np.array_equal(a.fit_errors, b.fit_errors)
    if b.job_allocated_hypernodes is not None:  # topology sessions: subJob.AllocatedHyperNode after the run
        assert a.job_allocated_hypernodes is not None
        assert np.array_equal(a.job_allocated_hypernodes, b.job_allocated_hypernodes)


@pytest.mark.parametrize("case", G.allocate_cases(), ids=lambda c: c.Name[:40])
def test_allocate_goldens(case, gpu, oracle_engine):
    snap = case.RegisterSession(G.allocate_tiers())
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()
    _assert_same(case.result, oracle_engine(snap))


def test_action_interface_like_the_reference(gpu):
    """test.RegisterSession(tiers, nil); test.Run([]framework.Action{allocate.New()}); test.CheckAll(i)"""
    from volcano_b200 import action
    case = G.allocate_cases()[3]
    case.RegisterSession(G.allocate_tiers())
    act = action.New()
    assert act.Name() == "allocate"
    case.Run([act])
    assert case.CheckAll() is None, case.CheckAll()


@pytest.mark.parametrize("case", G.fareshare_cases(), ids=lambda c: c.Name[:40])
def test_fareshare_goldens(case, gpu, oracle_engine):
    snap = case.RegisterSession(G.fareshare_tiers())
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()
    _assert_same(case.result, oracle_engine(snap))


@pytest.mark.parametrize("case,weights", G.nodeorder_cases(), ids=lambda c: getattr(c, "Name", "w")[:40])
def test_nodeorder_goldens(case, weights, gpu, oracle_engine):
    snap = case.RegisterSession(G.nodeorder_tiers(**weights))
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()
    _assert_same(case.result, oracle_engine(snap))


@pytest.mark.parametrize("case", G.proportion_cases(), ids=lambda c: c.Name[:40])
def test_proportion_goldens(case, gpu, oracle_engine):
    snap = case.RegisterSession(G.proportion_tiers())
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()
    _assert_same(case.result, oracle_engine(snap))


@pytest.mark.parametrize("case,nodes,scores", G.tdm_cases(), ids=lambda c: getattr(c, "Name", "x")[:40])
def test_tdm_goldens(case, nodes, scores, gpu):
    """tdm_test.go:107-270: predicate verdicts and scores of the tdm plugin through the dense pass."""
    from tests.test_oracle_golden import _check_tdm
    snap = case.RegisterSession(G.tdm_tiers())
    e = gpu.Engine(snap)
    e.upload()
    mask, score, _, _ = e.score_matrix()
    e.close()
    _check_tdm(snap, mask, score, nodes, scores)


@pytest.mark.parametrize("case,args,expected", G.nta_cases(), ids=lambda c: getattr(c, "Name", "x")[:40])
def test_nta_goldens(case, args, expected, gpu):
    """network_topology_aware_test.go:2011-2766, pods without a network topology: scores of the feasible nodes
    through the dense pass (only network-topology-aware registered, so the total IS the plugin's score)."""
    snap = case.RegisterSession(G.nta_tiers(args))
    e = gpu.Engine(snap)
    e.upload()
    mask, score, _, _ = e.score_matrix()
    e.close()
    t = snap.task_keys.index("ns1/p1")
    checked = 0
    for n, name in enumerate(snap.node_names):
        if (mask[t, n // 64] >> np.uint64(n % 64)) & np.uint64(1):
            assert abs(score[t, n] - expected.get(name, 0.0)) <= G.NTA_EPS, (name, score[t, n])
            checked += 1
    assert checked >= 6


def test_nta_soft_topology_allocate(gpu, oracle_engine):
    """Soft-mode topology job with an allocated hypernode and a running pod at open: LCA-tier scores, task-count
    tie term and allocated-hypernode tracking inside the commit kernel, against the oracle."""
    tc = G.nta_soft_allocate_case()
    snap = tc.RegisterSession(G.nta_soft_allocate_tiers())
    tc.Run(gpu.gpu_engine)
    _assert_same(tc.result, oracle_engine(snap))
    leaf = [tc.binds[f"c1/p{i}"].split("-")[0] for i in range(1, 7)]
    assert leaf.count("s3") == 3 and leaf.count("s4") == 3, leaf


@pytest.mark.parametrize("case", G.NTA_SOFT_ALLOCATE_CASES, ids=[c[0][24:70] for c in G.NTA_SOFT_ALLOCATE_CASES])
def test_allocate_with_network_topologies_soft(case, gpu, oracle_engine):
    """allocate_test.go:359-747, soft-mode rows of TestAllocateWithNetWorkTopologies through the CUDA engine."""
    tc = G.nta_soft_allocate_golden(case)
    snap = tc.RegisterSession(G.nta_soft_allocate_golden_tiers())
    tc.Run(gpu.gpu_engine)
    assert len(tc.binds) == tc.ExpectBindsNum, tc.binds
    if tc.ExpectBindMap:
        assert tc.CheckBind() is None, tc.CheckBind()
    _assert_same(tc.result, oracle_engine(snap))


@pytest.mark.parametrize("args,expected", G.BINPACK_CASES)
def test_binpack_goldens(args, expected, gpu):
    """binpack_test.go:100-238: exact scores through the dense pass (only binpack registered)."""
    from volcano_b200.snapshot import PluginOption
    from volcano_b200.uthelper import TestCommonStruct
    tc = TestCommonStruct(Name="binpack", **G.binpack_cluster())
    snap = tc.RegisterSession([[PluginOption.make("binpack", arguments=args, EnabledNodeOrder=True)]])
    e = gpu.Engine(snap)
    e.upload()
    mask, score, bs, bn = e.score_matrix()
    e.close()
    checked = 0
    for t, key in enumerate(snap.task_keys):
        for n, node in enumerate(snap.node_names):
            feasible = bool((mask[t, n // 64] >> np.uint64(n % 64)) & np.uint64(1))
            want = expected[key][node]
            if feasible:  # the dense pass scores feasible pairs only (allocate.predicate gates the rest)
                assert abs(score[t, n] - want) <= G.BINPACK_EPS, (key, node, score[t, n])
                checked += 1
    assert checked >= 4


ALLOC_CASES = [("tiny", 1), ("tiny", 2), ("tiny", 3), ("small", 1), ("cfg1", None), ("small", 7),
               # general kernel: FutureIdle gradient (Pipeline ops, KEEP visits), normalising TaintToleration scorer
               ("tiny_fut", 2), ("tiny_fut", None), ("small_fut_soft", None), ("small_fut_soft", 1), ("small_fut_soft", 2),
               ("small_soft", None), ("small_soft", 3),
               # two roles per job with different requests + TaskMinAvailable: role minima, predicate-error cache
               ("small_roles", None), ("small_roles", 5),
               # network-topology-aware: hypernode-level binpacking term, hyperNodeResourceCache updated per placement
               ("tiny_topo", None), ("tiny_topo", 3), ("small_topo", None), ("small_topo", 2),
               ("small_topo_fut_soft", None), ("small_topo_fut_soft", 4), ("small_topo_normal", None)]


@pytest.mark.parametrize("cfg,seed", ALLOC_CASES)
def test_allocate_vs_oracle(cfg, seed, gpu, oracle_engine):
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg, seed)
    res = gpu.gpu_engine(snap)
    ref = oracle_engine(snap, threads=4)
    _assert_same(res, ref)
    assert len(res.decisions) > 0


# ---- the backfill action (actions/backfill/backfill.go) on the state allocate left ----
@pytest.mark.parametrize("cfg,seed", [("tiny_bf", None), ("tiny_bf", 3), ("small_bf", None), ("small_bf", 5),
                                      ("small_soft_bf", None), ("small_soft_bf", 2),
                                      ("small_topo_bf", None), ("small_topo_bf", 4)])
def test_allocate_then_backfill_vs_oracle(cfg, seed, gpu, oracle_engine):
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg, seed)
    res = gpu.gpu_engine(snap)
    ref = oracle_engine(snap, threads=4)
    _assert_same(res, ref)
    assert res.backfill is not None and ref.backfill is not None
    _assert_same(res.backfill, ref.backfill)
    assert np.array_equal(res.backfill.decisions["score"], ref.backfill.decisions["score"])  # bit-equal fp64 totals
    assert len(res.backfill.decisions) > 0
    # every BestEffort task is either placed or carries fit errors; pod caps hold on every node after both actions
    assert len(res.backfill.decisions) + len(res.backfill.fit_errors) == snap.B
    placed = np.bincount(res.backfill.decisions["node"], minlength=snap.N)
    alloc_ops = res.decisions[res.decisions["kind"] == abi_mod().VC_OP_ALLOCATE]
    kept = np.isin(alloc_ops["visit"], np.nonzero(res.visits["outcome"] != abi_mod().VC_VISIT_DISCARD)[0])
    placed += np.bincount(alloc_ops["node"][kept], minlength=snap.N)
    pip = res.decisions[res.decisions["kind"] == abi_mod().VC_OP_PIPELINE]
    placed += np.bincount(pip["node"], minlength=snap.N)  # the predicates plugin counts pipelined pods too
    assert np.all(snap.n_pod_count + placed <= snap.n_max_tasks)


def abi_mod():
    from volcano_b200 import abi
    return abi


def test_backfill_alone_on_the_opening_state(gpu):
    """A cycle configured with backfill only: vc_backfill_run without vc_allocate_run starts from the opening node state."""
    from oracle.pyoracle import OracleSession
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot("small_bf", 11)
    e = gpu.Engine(snap)
    e.upload()
    res = e.backfill()
    with pytest.raises(gpu.VcError):  # once per session state
        e.backfill()
    e.close()
    o = OracleSession(snap, threads=4)
    dec, vis, fe = o.backfill()
    o.close()
    assert np.array_equal(res.decisions, dec) and np.array_equal(res.visits, vis) and np.array_equal(res.fit_errors, fe)


def test_backfill_pick_up_pending_tasks_golden(gpu):
    """backfill_test.go:39-154 TestPickUpPendingTasks through the C ABI: the session has no node, so every BestEffort task
    records fit errors - in pick order."""
    tc = G.backfill_pick_case()
    snap = tc.RegisterSession(G.backfill_pick_tiers(), actions=("allocate", "backfill"))
    res = gpu.gpu_engine(snap)
    assert res.backfill is not None and len(res.backfill.decisions) == 0
    assert [snap.backfill_task_keys[t] for t in res.backfill.fit_errors] == G.BACKFILL_PICK_EXPECTED
    assert [snap.job_names[j] for j in res.backfill.visits["job"]] == ["default/pg2", "default/pg1"]


def test_predicates_node_num_golden(gpu, oracle_engine):
    """predicates_test.go:194-259 TestNodeNum through test.Run([allocate.New(), backfill.New()])."""
    from volcano_b200 import action, backfill
    tc = G.predicates_node_num_case()
    snap = tc.RegisterSession(G.predicates_node_num_tiers(), actions=("allocate", "backfill"))
    tc.Run([action.New(), backfill.New()])
    assert tc.CheckBind() is None, tc.CheckBind()
    ref = oracle_engine(snap)
    _assert_same(tc.result, ref)
    _assert_same(tc.result.backfill, ref.backfill)


def test_backfill_action_interface(gpu, oracle_engine):
    """test.Run([]framework.Action{allocate.New(), backfill.New()}) with the reference's default plugin set: BestEffort pods
    are bound next to the regular ones; unsupported configurations fail loudly."""
    from volcano_b200 import action, backfill
    from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList
    from volcano_b200.snapshot import PluginOption, SchedulerConf
    from volcano_b200.uthelper import TestCommonStruct
    nodes = [BuildNode(f"n{i}", BuildResourceList("4", "8Gi", ("pods", "3"))) for i in range(3)]
    pods = [BuildPod("c1", f"w{i}", "", "Pending", BuildResourceList("1", "1Gi"), "pg1") for i in range(3)]
    pods += [BuildPod("c1", f"be{i}", "", "Pending", {}, "pg1") for i in range(4)]
    pods += [BuildPod("c1", f"xbe{i}", "", "Pending", {}, "pg2") for i in range(4)]
    pods += [BuildPod("c1", "xw0", "", "Pending", BuildResourceList("64", "1Gi"), "pg2")]  # never fits: pg2 stays unready
    tc = TestCommonStruct(Name="allocate+backfill", Nodes=nodes, Pods=pods, Queues=[BuildQueue("q1", 1, None)],
                          PodGroups=[BuildPodGroup("pg1", "c1", "q1", 2), BuildPodGroup("pg2", "c1", "q1", 5)])
    conf = SchedulerConf.default()
    snap = tc.RegisterSession(conf.tiers, actions=("allocate", "backfill"))
    assert snap.B == 8
    tc.Run([action.New(), backfill.New()])
    ref = oracle_engine(snap)
    _assert_same(tc.result, ref)
    _assert_same(tc.result.backfill, ref.backfill)
    # 9 pod slots, 3 taken by allocate. gang's JobOrderFn visits the unready pg2 (0 + 4 < 5) first: its four BestEffort
    # pods take four slots but stay Allocated in the session (ssn.JobReady false, no dispatch); pg1 is ready: two of its
    # BestEffort pods get the last two slots and are bound, the other two carry fit errors (pod-count predicate)
    bf = tc.result.backfill
    assert [snap.job_names[j] for j in bf.visits["job"]] == ["c1/pg2", "c1/pg1"]
    assert list(bf.visits["outcome"]) == [abi_mod().VC_VISIT_KEEP, abi_mod().VC_VISIT_COMMIT]
    assert len(bf.decisions) == 6 and [snap.backfill_task_keys[t] for t in bf.fit_errors] == ["c1/be2", "c1/be3"]
    assert sorted(tc.binds) == ["c1/be0", "c1/be1", "c1/w0", "c1/w1", "c1/w2"]
    assert bf.decisions["score"][-1] == 0.0  # one candidate left: taken without scoring (backfill.go:89-90)
    # feasible-node sampling carries on from the index allocate left
    tc2 = TestCommonStruct(Name="sampling", Nodes=nodes, Pods=pods, Queues=[BuildQueue("q1", 1, None)],
                           PodGroups=[BuildPodGroup("pg1", "c1", "q1", 2), BuildPodGroup("pg2", "c1", "q1", 5)])
    snap2 = tc2.RegisterSession(conf.tiers, actions=("allocate", "backfill"), percentage_nodes_to_find=50, min_nodes_to_find=1,
                                last_processed_node_index=2)
    tc2.Run([action.New(), backfill.New()])
    ref2 = oracle_engine(snap2)
    _assert_same(tc2.result, ref2)
    _assert_same(tc2.result.backfill, ref2.backfill)
    # the topology plugin: fine (a BestEffort pod touches no weighted hypernode resource) ...
    tc3 = TestCommonStruct(Name="nta", Nodes=nodes, Pods=pods, Queues=[BuildQueue("q1", 1, None)],
                           PodGroups=[BuildPodGroup("pg1", "c1", "q1", 2), BuildPodGroup("pg2", "c1", "q1", 5)])
    snap3 = tc3.RegisterSession([conf.tiers[0], conf.tiers[1] + [PluginOption.defaults("network-topology-aware")]],
                                actions=("allocate", "backfill"))
    tc3.Run([action.New(), backfill.New()])
    ref3 = oracle_engine(snap3)
    _assert_same(tc3.result, ref3)
    _assert_same(tc3.result.backfill, ref3.backfill)
    # ... unless "pods" itself is weighed: outside vc_backfill_run, fail loudly
    tc4 = TestCommonStruct(Name="unsupported", Nodes=nodes, Pods=pods, Queues=[BuildQueue("q1", 1, None)],
                           PodGroups=[BuildPodGroup("pg1", "c1", "q1", 2), BuildPodGroup("pg2", "c1", "q1", 5)])
    nta = PluginOption.defaults("network-topology-aware", {"hypernode.binpack.resources": "pods",
                                                           "hypernode.binpack.resources.pods": 3})
    tc4.RegisterSession([conf.tiers[0], conf.tiers[1] + [nta]], actions=("allocate", "backfill"))
    with pytest.raises(gpu.VcError) as ei:
        tc4.Run([action.New(), backfill.New()])
    assert ei.value.code == abi_mod().VC_EUNSUPPORTED


@pytest.mark.parametrize("cfg,seed", [("tiny", 1), ("small", 7), ("small_roles", None)])
def test_allocate_generic_kernel(cfg, seed, gpu, oracle_engine, monkeypatch):
    """The same sessions through k_commit (per-step full sweeps) instead of the incremental k_commit_fast."""
    from volcano_b200.synth import make_snapshot
    monkeypatch.setenv("VC_COMMIT_GENERIC", "1")
    snap = make_snapshot(cfg, seed)
    _assert_same(gpu.gpu_engine(snap), oracle_engine(snap, threads=2))


@pytest.mark.parametrize("cfg,seed", [("tiny", 1), ("small", 2), ("cfg1", None), ("small_fut_soft", None), ("small_soft", 1),
                                      ("tiny_topo", None), ("small_topo", 1), ("small_topo_fut_soft", None)])
def test_score_matrix_vs_oracle(cfg, seed, gpu):
    from oracle.pyoracle import OracleSession
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg, seed)
    e = gpu.Engine(snap)
    e.upload()
    mask, score, bs, bn = e.score_matrix()
    e.close()
    o = OracleSession(snap)
    omask, oscore, obs, obn = o.score_matrix()
    o.close()
    assert np.array_equal(mask, omask)
    assert np.array_equal(bn, obn)
    assert np.allclose(score, oscore, rtol=0, atol=SCORE_TOL)
    assert np.allclose(bs, obs, rtol=0, atol=SCORE_TOL)
    assert np.array_equal(score, oscore), "scores are expected to be bit-identical"


def test_deserved_vs_oracle(gpu):
    from oracle.pyoracle import OracleSession
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot("small", 3)
    e = gpu.Engine(snap)
    e.upload()
    des, share = e.queue_deserved()
    e.close()
    o = OracleSession(snap)
    odes, oshare = o.queue_deserved()
    o.close()
    assert np.array_equal(des, odes) and np.array_equal(share, oshare)


@pytest.mark.parametrize("cfg", ["cfg2", "cfg3", "cfg4"])
def test_full_size_properties(cfg, gpu):
    """BASELINE configs[1..3] at full size (10k x 100k; + drf / proportion over 16 queues; 50k x 1M with the HyperNode
    tree and network-topology-aware): size-independent properties — every decision respects capacity, re-running is
    idempotent, gang minAvailable holds for every committed job."""
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg)
    e = gpu.Engine(snap)
    e.upload()
    r1 = e.allocate()
    r2 = e.allocate()
    e.close()
    assert np.array_equal(r1.decisions, r2.decisions) and np.array_equal(r1.visits, r2.visits)
    dec = r1.decisions
    assert len(np.unique(dec["task"])) == len(dec)  # a task is placed at most once
    used = snap.n_used.copy()
    np.add.at(used.T, dec["node"], snap.t_resreq.T[dec["task"]])
    assert (used <= snap.n_allocatable + 0.1).all()  # no node over-committed on any dimension
    # gang: committed allocations per job >= minAvailable
    committed = r1.visits["outcome"][dec["visit"]] == 0
    per_job = np.bincount(snap.t_job[dec["task"][committed]], minlength=snap.J)
    jobs_committed = np.unique(r1.visits["job"][r1.visits["outcome"] == 0])
    assert (per_job[jobs_committed] >= snap.j_min_available[jobs_committed]).all()


def _host_threads():
    import os
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    return max(1, min(16, n))  # the reference runs 16 workers per task (util/predicate_helper.go:133)


FULL_SIZE = [("cfg2", "fast"), ("cfg2", "fast_norun"), ("cfg2", "generic"), ("cfg2", "sampling"), ("cfg3", "fast"), ("cfg3", "generic"),
             ("cfg2_fut", "fast"), ("cfg2_fut_tight", "fast"), ("cfg3_fut", "fast"), ("cfg2_soft", "fast"), ("cfg2_fut_soft", "fast")]


@pytest.mark.parametrize("cfg,mode", FULL_SIZE, ids=[f"{c}-{m}" for c, m in FULL_SIZE])
def test_full_size_vs_oracle(cfg, mode, gpu, oracle_engine):
    """BASELINE configs[1] / [2] at FULL size (10k nodes x 100k tasks) — the configuration bench.py measures: every
    decision (task, node, kind, visit, fp64 score), every visit outcome and every fit error against the oracle
    (actions/allocate/allocate.go:283-348, :558-694). Modes: the incremental kernel with and without run-length
    batches, the general kernel (VC_COMMIT_GENERIC), and the reference's default feasible-node sampling
    (percentage-nodes-to-find=0 -> adaptive 5 %, util/scheduler_helper.go:54-73)."""
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg)
    threads = _host_threads()
    if mode == "sampling":
        snap.conf.percentage_nodes_to_find = 0
        threads = 1  # the single-worker reading of the early-stop loop
    gpu.debug_option("VC_COMMIT_GENERIC", 1 if mode == "generic" else 0)
    gpu.debug_option("VC_COMMIT_NORUN", 1 if mode == "fast_norun" else 0)
    try:
        res = gpu.gpu_engine(snap)
    finally:
        gpu.debug_option("VC_COMMIT_GENERIC", 0)
        gpu.debug_option("VC_COMMIT_NORUN", 0)
    ref = oracle_engine(snap, threads=threads)
    assert len(ref.decisions) > 90_000 or mode == "sampling" or "fut" in cfg
    if "fut" in cfg or "soft" in cfg:  # Releasing resources / PreferNoSchedule taints: the incremental kernel's FUT / SOFT instances
        assert res.stats["commit_kernel"] == 1, res.stats  # VC_KERNEL_INCREMENTAL
    if "fut" in cfg:
        assert (ref.decisions["kind"] == 1).sum() > (1000 if "tight" in cfg else 0)
    _assert_same(res, ref)
    assert np.array_equal(res.decisions["score"], ref.decisions["score"]), "scores are expected to be bit-identical"


def test_cfg4_sampled_replay(gpu):
    """BASELINE config 4 (50k nodes x 1M tasks, 3-tier HyperNode tree, network-topology-aware, drf + proportion over 16
    queues) — BASELINE.md section 3: the GPU's decision list is replayed through the oracle session and every 100th
    decision (1 %) is re-derived on the state reached so far: feasible nodes, prioritizeNodes arg-max, fp64 score."""
    from oracle.pyoracle import OracleSession
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot("cfg4")
    res = gpu.gpu_engine(snap)
    assert len(res.decisions) > 500_000
    o = OracleSession(snap, threads=_host_threads())
    bad, first, checked = o.replay_check(res.decisions, res.visits, 100, 37)
    o.close()
    assert checked >= len(res.decisions) // 100 - 1
    assert bad == 0, f"{bad} of {checked} sampled decisions differ, first at index {first}"


SAMPLING_CASES = [("tiny", 1, 50, 10, 0), ("tiny", 2, 20, 5, 17), ("small", 7, 0, 100, 0), ("small", 3, 30, 50, 333),
                  ("tiny_fut", 2, 40, 8, 5), ("small_fut_soft", None, 25, 30, 0), ("small_roles", None, 35, 20, 11),
                  ("small_topo", None, 30, 40, 100), ("small_topo_fut_soft", 4, 50, 20, 7), ("cfg1", None, 0, 20, 0)]


@pytest.mark.parametrize("cfg,seed,pct,min_nodes,start", SAMPLING_CASES)
def test_feasible_node_sampling_vs_oracle(cfg, seed, pct, min_nodes, start, gpu, oracle_engine):
    """util.PredicateNodes with percentage-nodes-to-find < 100 (predicate_helper.go:43-140, scheduler_helper.go:54-73)
    in its single-worker reading: stop after numNodesToFind feasible nodes, rotating start index carried across tasks."""
    from oracle.pyoracle import OracleSession
    from oracle import pyoracle
    from volcano_b200.synth import make_snapshot
    snap = make_snapshot(cfg, seed)
    snap.conf.percentage_nodes_to_find = pct
    snap.conf.min_nodes_to_find = min_nodes
    snap.conf.last_processed_node_index = start
    res = gpu.gpu_engine(snap)
    o = OracleSession(snap, threads=1)
    dec, vis, fe = o.allocate()
    last = pyoracle.lib().vco_last_processed_node_index(o.h)
    o.close()
    assert np.array_equal(res.decisions, dec) and np.array_equal(res.visits, vis) and np.array_equal(res.fit_errors, fe)
    assert res.stats["last_processed_node_index"] == last
    assert len(dec) > 0


def _assert_same_evict(a, b):
    assert (a is None) == (b is None)
    if a is None:
        return
    assert np.array_equal(a.visits, b.visits), (a.visits, b.visits)
    for f in ("task", "node", "kind", "visit"):
        assert np.array_equal(a.decisions[f], b.decisions[f]), f


@pytest.mark.parametrize("case", G.preempt_cases(), ids=lambda c: c.Name[:50])
def test_preempt_goldens(case, gpu, oracle_engine):
    """actions/preempt/preempt_test.go:54-425 TestPreempt through vc_preempt_run; statements compared with the oracle's."""
    snap = case.RegisterSession(G.preempt_tiers(), actions=("preempt",))
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()
    _assert_same_evict(case.result.preempt, oracle_engine(snap).preempt)


@pytest.mark.parametrize("plugins,case", G.reclaim_cases(), ids=lambda c: getattr(c, "Name", "p")[:50])
def test_reclaim_goldens(plugins, case, gpu, oracle_engine):
    """actions/reclaim/reclaim_test.go:47-388 TestReclaim through vc_reclaim_run."""
    snap = case.RegisterSession(G.reclaim_tiers(plugins), actions=("reclaim",))
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()
    _assert_same_evict(case.result.reclaim, oracle_engine(snap).reclaim)


def test_preempt_action_interface(gpu):
    """test.Run([]framework.Action{preempt.New()}) like the reference's TestPreempt."""
    from volcano_b200 import preempt
    case = G.preempt_cases()[3]
    case.RegisterSession(G.preempt_tiers(), actions=("preempt",))
    act = preempt.New("preempt")
    assert act.Name() == "preempt"
    case.Run([act])
    assert case.CheckAll() is None, case.CheckAll()


def test_cfg5_cycle_vs_oracle(gpu, oracle_engine):
    """BASELINE configs[4] at a reduced size (1 000 nodes near capacity, ~1 500 pending tasks, 8 queues): the cycle
    allocate -> preempt -> reclaim through the C ABI, every decision and statement against the oracle."""
    from volcano_b200.synth import make_cfg5
    snap = make_cfg5(seed=77, n_nodes=1000, n_pending=1500, n_queues=8, utilisation=0.9)
    res = gpu.gpu_engine(snap)
    ref = oracle_engine(snap, threads=_host_threads())
    _assert_same(res, ref)
    _assert_same_evict(res.preempt, ref.preempt)
    _assert_same_evict(res.reclaim, ref.reclaim)
    assert (ref.preempt.decisions["kind"] == 2).sum() + (ref.reclaim.decisions["kind"] == 2).sum() > 10


def test_cfg5_cycle_10k_vs_oracle(gpu, oracle_engine):
    """BASELINE configs[4] at its full node count (10 000 nodes near capacity, 8 queues) with ~1 500 pending tasks: each
    thread of the cached pick kernel owns ~10 nodes, so every hand-out repairs a lane's list by rescanning several nodes."""
    from volcano_b200.synth import make_cfg5
    snap = make_cfg5(seed=77, n_nodes=10_000, n_pending=1500, n_queues=8, utilisation=0.9)
    res = gpu.gpu_engine(snap)
    ref = oracle_engine(snap, threads=_host_threads())
    _assert_same(res, ref)
    _assert_same_evict(res.preempt, ref.preempt)
    _assert_same_evict(res.reclaim, ref.reclaim)
    assert (ref.preempt.decisions["kind"] == 2).sum() > 100 and (ref.reclaim.decisions["kind"] == 2).sum() > 100


def test_evict_past_the_pick_cache_vs_oracle(gpu, oracle_engine):
    """More than 25 600 nodes: the candidates' keys no longer fit in shared memory and production hands out candidates
    with k_evict_pick_big. A small pending set keeps the oracle quick."""
    from volcano_b200.synth import make_cfg5
    snap = make_cfg5(seed=5, n_nodes=26_000, n_pending=200, n_queues=8, utilisation=0.6)
    assert snap.N * 8 > 200 * 1024
    res = gpu.gpu_engine(snap)
    ref = oracle_engine(snap, threads=_host_threads())
    _assert_same(res, ref)
    _assert_same_evict(res.preempt, ref.preempt)
    _assert_same_evict(res.reclaim, ref.reclaim)
    assert (ref.preempt.decisions["kind"] == 2).sum() + (ref.reclaim.decisions["kind"] == 2).sum() > 10


def _victims_cluster(n_victims):
    """One node full of single-core pods of a low-priority job, and a starving high-priority job of the same queue whose
    one pod needs n_victims of those cores back."""
    from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList
    from volcano_b200.snapshot import PluginOption
    from volcano_b200.uthelper import TestCommonStruct
    cores = n_victims + 1
    node = BuildNode("n0", BuildResourceList(str(cores), f"{cores}Gi", ("pods", str(cores + 10))))
    low = BuildPodGroup("low", "ns", "q", 1, None, "Running")
    high = BuildPodGroup("high", "ns", "q", 1, None, "Inqueue")
    low.priority, high.priority = 1, 100
    pods = [BuildPod("ns", f"low-{k}", "n0", "Running", BuildResourceList("1", "1Gi"), "low", {}) for k in range(cores)]
    pods.append(BuildPod("ns", "high-0", "", "Pending", BuildResourceList(str(n_victims), "1Gi"), "high", {}))
    tc = TestCommonStruct(Name=f"victims{n_victims}", Nodes=[node], Pods=pods, PodGroups=[low, high], Queues=[BuildQueue("q", 1, None)])
    tiers = [[PluginOption.defaults("priority"), PluginOption.defaults("gang"), PluginOption.defaults("conformance")]]
    return tc.RegisterSession(tiers, actions=("preempt",))


def test_evict_max_victims(gpu, oracle_engine):
    """EV_MAX_VICTIMS: a preemptor that needs exactly 256 victims on one node matches the oracle; one that needs 257 is
    refused with VC_EUNSUPPORTED instead of overrunning the apply command."""
    snap = _victims_cluster(256)
    res, ref = gpu.gpu_engine(snap), oracle_engine(snap)
    _assert_same_evict(res.preempt, ref.preempt)
    assert (ref.preempt.decisions["kind"] == 2).sum() == 256 and (ref.preempt.decisions["kind"] == 1).sum() == 1
    snap = _victims_cluster(257)
    assert (oracle_engine(snap).preempt.decisions["kind"] == 2).sum() == 257
    with pytest.raises(gpu.VcError) as ei:
        gpu.gpu_engine(snap)
    assert ei.value.code == abi_mod().VC_EUNSUPPORTED


def test_nominated_node_vs_oracle(gpu, oracle_engine):
    """Pod.Status.NominatedNodeName (actions/allocate/allocate.go:624-634): the nominated node is tried first, alone; parity
    with the oracle in the full-evaluation mode and with feasible-node sampling (where the one-node PredicateNodes call
    resets util.lastProcessedNodeIndex), on the general commit kernel such sessions take."""
    from tests.test_oracle_golden import _nominated_cluster
    for args in (("n2",), ("n0", "8"), ("gone",), ("n2", "4", 34), ("n1", "4", 67)):
        tc = _nominated_cluster(*args)
        res = gpu.gpu_engine(tc.snap)
        ref = oracle_engine(tc.snap)
        _assert_same(res, ref)
        if (tc.snap.t_nominated >= 0).any():
            assert res.stats["commit_kernel"] == 0  # VC_KERNEL_GENERAL
        from oracle.pyoracle import OracleSession
        from oracle import pyoracle
        o = OracleSession(tc.snap, threads=1)
        o.allocate()
        assert res.stats["last_processed_node_index"] == pyoracle.lib().vco_last_processed_node_index(o.h), args
        o.close()
