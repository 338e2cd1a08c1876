"""One snapshot handle through a sequence of sessions of one shape (one vc_dims) that grow and then shrink every
sub-allocated device slab: the running-task table of the evicting actions, the pdb table, the topology-aware dry run's
slab, the areas of hypernode binpacking, the backfill slab, and the dense pass materialised after an evicting action.
Every run equals the same session on a fresh handle bit for bit: decisions, visits, fit errors and
lastProcessedNodeIndex (and the dense pass's mask, scores and best nodes)."""
import numpy as np
import pytest

from volcano_b200.api import (BuildHyperNode, BuildNode, BuildPDB, BuildPod, BuildPodGroup, BuildQueue,
                              BuildResourceList)
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct

pytestmark = pytest.mark.gpu

N_NODES = 16
EVICT = ("allocate", "preempt", "reclaim")
BACKFILL = ("allocate", "backfill")


def _session(run_per_node, n_pdb=1, topo_aware=False, binpack=False, n_besteffort=0, actions=EVICT):
    """16 nodes of 8 CPUs under a tree of 4-node leaves; job `low` (q0) runs `run_per_node` 2-CPU pods on every node and
    `other` (q1) one pod on each of the first four; `high` (q0, priority 1000) needs 7 CPUs per pod, so it preempts, and
    `starve` (q1) 5 CPUs per pod, so it reclaims. `n_pdb` PDBs over the running pods of `low`, `n_besteffort`
    BestEffort pods in `starve`. The running pods, PDBs and options leave vc_dims as they are."""
    nodes = [BuildNode(f"n{i:02d}", BuildResourceList("8", "16G", ("pods", "110"))) for i in range(N_NODES)]
    queues = [BuildQueue("q0", 1), BuildQueue("q1", 1)]
    pgs = [BuildPodGroup("low", "ns", "q0", 1, None, "Running"), BuildPodGroup("other", "ns", "q1", 1, None, "Running"),
           BuildPodGroup("high", "ns", "q0", 1, None, "Inqueue"), BuildPodGroup("starve", "ns", "q1", 1, None, "Inqueue")]
    pgs[2].priority = 1000
    pods = []
    for i, n in enumerate(nodes):
        for k in range(run_per_node):
            pods.append(BuildPod("ns", f"low-{i}-{k}", n.name, "Running", BuildResourceList("2", "1G"), "low",
                                 {"volcano.sh/preemptable": "true", "app": "a" if k % 2 == 0 else "b"}))
        if i < 4:
            pods.append(BuildPod("ns", f"other-{i}", n.name, "Running", BuildResourceList("1", "1G"), "other",
                                 {"volcano.sh/preemptable": "true", "app": "b"}))
    pods += [BuildPod("ns", f"high-{k}", "", "Pending", BuildResourceList("7", "2G"), "high") for k in range(4)]
    pods += [BuildPod("ns", f"starve-{k}", "", "Pending", BuildResourceList("5", "2G"), "starve") for k in range(3)]
    pods += [BuildPod("ns", f"be-{k}", "", "Pending", {}, "starve") for k in range(n_besteffort)]
    leaves = [BuildHyperNode(f"leaf{h}", 1, [(nodes[m].name, "Node") for m in range(4 * h, 4 * h + 4)]) for h in range(4)]
    tree = leaves + [BuildHyperNode("midA", 2, [("leaf0", "HyperNode"), ("leaf1", "HyperNode")]),
                     BuildHyperNode("midB", 2, [("leaf2", "HyperNode"), ("leaf3", "HyperNode")]),
                     BuildHyperNode("root", 3, [("midA", "HyperNode"), ("midB", "HyperNode")])]
    pdbs = [BuildPDB("ns", f"pdb{i}", [{"app": "a"}, {"app": "b"}][i % 2], 1 + i % 3) for i in range(n_pdb)]
    nta = {"weight": 10, "hypernode.binpack.cpu": 5, "hypernode.binpack.memory": 1,
           "hypernode.binpack.normal-pod.enable": binpack, "hypernode.binpack.normal-pod.fading": 0.5}
    tiers = [[PluginOption.defaults(n) for n in ("priority", "gang", "conformance", "pdb")],
             [PluginOption.defaults(n) for n in ("drf", "proportion", "predicates", "nodeorder")] +
             [PluginOption.defaults("network-topology-aware", nta)]]
    preempt = {"enableTopologyAwarePreemption": topo_aware, "minCandidateNodesPercentage": 10,
               "minCandidateNodesAbsolute": 1, "maxCandidateNodesAbsolute": 100}
    tc = TestCommonStruct(Name="reuse", Nodes=nodes, Pods=pods, PodGroups=pgs, Queues=queues, HyperNodes=tree, PDBs=pdbs)
    return tc.RegisterSession(tiers, actions=actions, configurations={"preempt": preempt}, preempt_seed=7, now_ns=10 ** 18)


# (session, materialise the dense pass after the actions): each slab grows, then shrinks
SEQUENCE = [
    (dict(run_per_node=1), False),
    (dict(run_per_node=3, n_pdb=4), False),                                   # running-task table and pdb table grow
    (dict(run_per_node=3, n_pdb=4, topo_aware=True), False),                  # topology-aware slab
    (dict(run_per_node=3, n_pdb=4, topo_aware=True, binpack=True), False),    # ... and the binpacking areas
    (dict(run_per_node=1, topo_aware=True, binpack=True), False),             # every one of them shrinks
    (dict(run_per_node=2, n_pdb=2, binpack=True), False),                     # binpacking without the dry run
    (dict(run_per_node=1), False),                                            # binpacking off again
    (dict(run_per_node=1, n_besteffort=200, actions=BACKFILL), False),        # backfill slab
    (dict(run_per_node=1, n_besteffort=1200, actions=BACKFILL), False),
    (dict(run_per_node=1, n_besteffort=30, actions=BACKFILL), False),
    (dict(run_per_node=2, n_pdb=2, binpack=True), True),                      # dense pass after the evicting actions
    (dict(run_per_node=3, n_pdb=3, topo_aware=True), True),
    (dict(run_per_node=1), True),
]


def _run(e, snap, dense):
    e.upload(snap)
    out = [(a, getattr(e, a)()) for a in snap.actions]
    if dense:
        out.append(("dense", e.score_matrix()))
    return out


def _same(a, b, what):
    assert [x for x, _ in a] == [y for y, _ in b], what
    for (name, x), (_, y) in zip(a, b):
        if name == "dense":
            for u, v in zip(x, y):
                assert u.tobytes() == v.tobytes(), (what, name)
            continue
        for f in x.decisions.dtype.names:
            assert x.decisions[f].tobytes() == y.decisions[f].tobytes(), (what, name, f)
        for f in x.visits.dtype.names:
            assert x.visits[f].tobytes() == y.visits[f].tobytes(), (what, name, f)
        assert x.fit_errors.tobytes() == y.fit_errors.tobytes(), (what, name)
        assert x.stats["last_processed_node_index"] == y.stats["last_processed_node_index"], (what, name)


def test_sessions_of_one_shape_on_one_handle():
    from volcano_b200 import abi, engine
    engine.init(0)
    snaps = [(_session(**kw), dense) for kw, dense in SEQUENCE]
    dims = [bytes(s.dims()) for s, _ in snaps]
    assert all(d == dims[0] for d in dims), "the sessions must share one vc_dims"
    evicted = 0
    reused = engine.Engine(snaps[0][0])
    try:
        for step, (snap, dense) in enumerate(snaps):
            got = _run(reused, snap, dense)
            fresh = engine.Engine(snap)
            try:
                want = _run(fresh, snap, dense)
            finally:
                fresh.close()
            _same(got, want, (step, SEQUENCE[step]))
            evicted += sum(int((r.decisions["kind"] == abi.VC_OP_EVICT).sum()) for a, r in got if a in ("preempt", "reclaim"))
    finally:
        reused.close()
    assert evicted > 0
