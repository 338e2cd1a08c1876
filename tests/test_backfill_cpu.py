"""CPU-side checks of the backfill action's host logic and of its oracle (actions/backfill/backfill.go): what the encoder
hands to vc_snapshot_set_backfill, and the semantics the CUDA path is compared against on the GPU box."""
import numpy as np

from oracle.pyoracle import OracleSession
from volcano_b200 import abi
from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList
from volcano_b200.snapshot import SchedulerConf
from volcano_b200.synth import make_snapshot
from volcano_b200.uthelper import AllocateResult, TestCommonStruct


def _cluster():
    nodes = [BuildNode(f"n{i}", BuildResourceList("4", "8Gi", ("pods", "3"))) for i in range(3)]
    pods = [BuildPod("c1", f"w{i}", "", "Pending", BuildResourceList("1", "1Gi"), "pg1") for i in range(3)]
    pods += [BuildPod("c1", f"be{i}", "", "Pending", {}, "pg1") for i in range(4)]
    pods += [BuildPod("c1", f"xbe{i}", "", "Pending", {}, "pg2") for i in range(4)]
    pods += [BuildPod("c1", "xw0", "", "Pending", BuildResourceList("64", "1Gi"), "pg2")]
    return TestCommonStruct(Name="allocate+backfill", Nodes=nodes, Pods=pods, Queues=[BuildQueue("q1", 1, None)],
                            PodGroups=[BuildPodGroup("pg1", "c1", "q1", 2), BuildPodGroup("pg2", "c1", "q1", 5)])


def test_encoder_splits_besteffort_tasks():
    tc = _cluster()
    snap = tc.RegisterSession(SchedulerConf.default().tiers, actions=("allocate", "backfill"))
    assert snap.T == 4 and snap.B == 8
    assert snap.backfill_task_keys == [f"c1/be{i}" for i in range(4)] + [f"c1/xbe{i}" for i in range(4)]
    assert list(snap.j_pending_besteffort) == [4, 4]
    pods_dim = snap.dim_names.index("pods")
    assert np.all(snap.b_resreq[pods_dim] == 1.0) and snap.b_resreq.sum() == 8.0  # Resreq = pods:1 only
    assert np.all(snap.b_k8s_nonzero_req[0] == 100.0) and np.all(snap.b_k8s_nonzero_req[1] == 200.0 * 2**20)
    bt = snap.backfill_tasks()
    assert isinstance(bt, abi.vc_tasks)
    # a session without BestEffort pods hands nothing over
    assert make_snapshot("tiny").backfill_tasks() is None


def test_backfill_semantics_on_the_oracle(oracle_engine):
    """Order (gang's JobOrderFn puts the unready job first), no resource fit but the pod-count predicate, one-candidate
    shortcut, dispatch only when ssn.JobReady holds."""
    tc = _cluster()
    snap = tc.RegisterSession(SchedulerConf.default().tiers, actions=("allocate", "backfill"))
    tc.Run(oracle_engine)
    bf = tc.result.backfill
    assert [snap.job_names[j] for j in bf.visits["job"]] == ["c1/pg2", "c1/pg1"]
    assert list(bf.visits["outcome"]) == [abi.VC_VISIT_KEEP, abi.VC_VISIT_COMMIT]
    assert len(bf.decisions) == 6 and [snap.backfill_task_keys[t] for t in bf.fit_errors] == ["c1/be2", "c1/be3"]
    assert sorted(tc.binds) == ["c1/be0", "c1/be1", "c1/w0", "c1/w1", "c1/w2"]
    assert bf.decisions["score"][-1] == 0.0
    per_node = np.bincount(np.concatenate([tc.result.decisions["node"], bf.decisions["node"]]), minlength=3)
    assert list(per_node) == [3, 3, 3]


def test_backfill_alone_and_synthetic_configs():
    snap = make_snapshot("tiny_bf")
    assert snap.B == 150 and "backfill" in snap.actions
    o = OracleSession(snap)
    order = o.backfill_pick_order()
    assert sorted(order) == list(range(snap.B))  # every job is valid and not Pending: all tasks are picked up
    jobs = snap.b_job[order]
    assert len(set(zip(jobs[:-1], jobs[1:])) - {(a, a) for a in jobs}) == len(set(jobs)) - 1  # one contiguous run per job
    dec, vis, fe = o.backfill()  # no allocate before: the opening state
    o.close()
    assert len(dec) + len(fe) == snap.B and vis["n_ops"].sum() == len(dec)
    res = AllocateResult(dec, vis, fe)
    assert np.all(np.diff(res.decisions["visit"]) >= 0)


def _pending_phase_cluster():
    """Two PodGroups still in phase Pending (no enqueue action has promoted them), BestEffort pods only in pg2."""
    nodes = [BuildNode("n0", BuildResourceList("4", "8Gi", ("pods", "8")))]
    pods = [BuildPod("c1", "w0", "", "Pending", BuildResourceList("1", "1Gi"), "pg1")]
    pods += [BuildPod("c1", f"be{i}", "", "Pending", {}, "pg2") for i in range(2)]
    pods += [BuildPod("c1", "w1", "", "Pending", BuildResourceList("1", "1Gi"), "pg2")]
    return TestCommonStruct(Name="pending phase", Nodes=nodes, Pods=pods, Queues=[BuildQueue("q1", 1, None)],
                            PodGroups=[BuildPodGroup("pg1", "c1", "q1", 1, None, "Pending"),
                                       BuildPodGroup("pg2", "c1", "q1", 1, None, "Pending")])


def test_pending_podgroups_without_the_enqueue_action(oracle_engine):
    """allocate.go:154-164: with no enqueue action configured buildAllocateContext rewrites the phase of every Pending
    PodGroup to Inqueue, so the backfill action that follows (backfill.go:124 job.IsPending()) places their BestEffort
    pods; with enqueue configured both actions skip such jobs."""
    tc = _pending_phase_cluster()
    snap = tc.RegisterSession(SchedulerConf.default().tiers, actions=("allocate", "backfill"))
    assert snap.conf.enqueue_action_enabled == 0 and (snap.j_flags & abi.VC_JOB_PENDING_PHASE).all()
    tc.Run(oracle_engine)
    assert sorted(tc.binds) == ["c1/be0", "c1/be1", "c1/w0", "c1/w1"]
    tc = _pending_phase_cluster()
    tc.RegisterSession(SchedulerConf.default().tiers, actions=("enqueue", "allocate", "backfill"))
    tc.Run(oracle_engine)
    assert tc.binds == {}
    # backfill alone (allocate did not run, nothing rewrote the phase): Pending jobs are skipped
    tc = _pending_phase_cluster()
    snap = tc.RegisterSession(SchedulerConf.default().tiers, actions=("backfill",))
    o = OracleSession(snap)
    assert len(o.backfill_pick_order()) == 0
    o.close()


def test_sampling_that_finds_no_node_on_the_oracle():
    """min_nodes_to_find 0 and 10 nodes at 5 %: numNodesToFind is 0 (util/scheduler_helper.go:54-73), so every scan of
    util.PredicateNodes finds nothing - allocate places no task and backfill lists every BestEffort task in fit_errors,
    and the single-worker scan leaves lastProcessedNodeIndex where it was. The library refuses such a session."""
    import dataclasses

    from oracle import pyoracle
    from volcano_b200.synth import CONFIGS
    snap = make_snapshot(dataclasses.replace(CONFIGS["tiny_bf"], n_nodes=10, n_tasks=40, n_besteffort=20))
    snap.conf.percentage_nodes_to_find, snap.conf.min_nodes_to_find, snap.conf.last_processed_node_index = 5, 0, 3
    L = pyoracle.lib()
    assert L.vco_num_feasible_nodes(10, 5, 0, snap.conf.min_percentage_nodes_to_find) == 0
    o = OracleSession(snap)
    dec, _, fe = o.allocate()
    assert len(dec) == 0 and len(fe) > 0
    order = o.backfill_pick_order()
    dec, vis, fe = o.backfill()
    assert len(order) > 0 and len(dec) == 0 and sorted(fe) == sorted(order)
    assert L.vco_last_processed_node_index(o.h) == 3
    o.close()
    # one more node, or a minimum of 1, and the same session places pods again
    snap.conf.min_nodes_to_find = 1
    o = OracleSession(snap)
    o.allocate()
    assert len(o.backfill()[0]) > 0
    o.close()


def test_besteffort_jobs_knob():
    """SynthConfig.besteffort_jobs puts every BestEffort pod into that many jobs; the default leaves the snapshot as it
    was, and the regular part of the session never depends on it."""
    import dataclasses

    from volcano_b200.synth import CONFIGS
    base = CONFIGS["small_bf"]
    assert base.besteffort_jobs == 0
    a = make_snapshot(base)
    b = make_snapshot(dataclasses.replace(base, besteffort_jobs=0))
    for k, v in a.__dict__.items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(v, getattr(b, k)), k
    for k, want in ((1, 1), (3, 3)):
        c = make_snapshot(dataclasses.replace(base, besteffort_jobs=k))
        assert len(np.unique(c.b_job)) == want and c.B == base.n_besteffort
        assert np.all(np.diff(c.b_job) >= 0)
        assert (c.j_pending_besteffort > 0).sum() == want and c.j_pending_besteffort.sum() == c.B
        for name in ("t_resreq", "t_job", "t_klass", "n_idle", "n_label_bits", "c_selector", "j_queue"):
            assert np.array_equal(getattr(a, name), getattr(c, name)), name
