"""Hand-derived sessions for preempt and reclaim under feasible-node sampling. Each builder returns the snapshot and
what the reference does with it (derived in the builder's docstring from preempt.go, reclaim.go, predicate_helper.go
and scheduler_helper.go): the PredicateNodes calls of the evicting actions in order, the index each action leaves, and
the statements of the evicting actions. Node names n0.. are NodeList positions."""
from __future__ import annotations

from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList
from volcano_b200.snapshot import PluginOption, PreemptArguments
from volcano_b200.uthelper import TestCommonStruct

PREEMPTABLE = {"volcano.sh/preemptable": "true"}


def _pod(name, node, prio=None, role=None, zone=None, never=False, labels=None):
    lab = dict(labels or {})
    if role is not None:
        lab["volcano.sh/task-spec"] = role
    p = BuildPod("ns", name, node, "Running" if node else "Pending", BuildResourceList("2", "1G"), name.split("-")[0], lab,
                 {"zone": zone} if zone else {})
    if prio is not None:
        p.priority = prio
    if never:
        p.preemption_policy = "Never"
    return p


def chain_case():
    """Five 1-CPU nodes: n1 and n3 labelled zone=a, n4 zone=d, n0 and n2 zone=b. One starving job "j" (minMember 1,
    Inqueue) of four 2-CPU pending pods, so nothing fits anywhere and no pod runs: every preemptor and reclaimer fails.
    percentage 50, min-nodes-to-find 1: numNodesToFind(5) = 2, (2) = 1, (1) = 1 (scheduler_helper.go:54-73), sampling on.
    lastProcessedNodeIndex 7 (>= N). Actions allocate, preempt, reclaim. Task order (priority): c (30, role x, zone=a),
    f (20, role v, zone=d), a (10, role y), e (5, role w, PreemptionPolicy Never).

    allocate: NeedContinueAllocating holds (minMember 1 < 4 tasks), so all four fail the predicate on every node, each an
    entry with node errors (four roles). Every failing scan visits all 5 nodes: the index becomes (7 + 5) % 5 = 2.
    Filtered lists (FilterOutUnschedulableAndUnresolvableNodesForTask): c [n1, n3] (P 2), f [n4] (P 1), a every node (P 5).
    preempt, inter-job phase (preempt.go:163-243), every task while the job starves:
      c: start 2, list[2 % 2] = n1 passes: [n1], processed 1, index (2 + 1) % 2 = 1;
      f: start 1 >= P = 1, a full scan (P <= numNodesToFind): [n4], processed 1, index (1 + 1) % 1 = 0;
      a: start 0: n0, n1: [n0, n1], processed 2, index 2;
      e: taskEligibleToPreempt refuses it (preempt.go:436-441) before PredicateNodes: no call.
    The job is not pipelined: discard. Intra-job phase (preempt.go:246-280): the first task c fails, the loop breaks:
      c: start 2, list[0] = n1: [n1], processed 1, index (2 + 1) % 2 = 1.
    preempt leaves 1. reclaim (reclaim.go:120-180), every task while the job starves:
      c: start 1, list[1] = n3: [n3], processed 1, index (1 + 1) % 2 = 0;
      f: [n4], processed 1, index 0;
      a: start 0: [n0, n1], processed 2, index 2;
      e: PreemptionPolicy Never (reclaim.go:140-143): no call.
    reclaim leaves 2."""
    nodes = [BuildNode(f"n{i}", BuildResourceList("1", "1G", ("pods", "10")), {"zone": z})
             for i, z in enumerate("babad")]
    pods = [_pod("j-c", "", 30, "x", "a"), _pod("j-f", "", 20, "v", "d"), _pod("j-a", "", 10, "y"),
            _pod("j-e", "", 5, "w", never=True)]
    tc = TestCommonStruct(Name="samp-chain", Nodes=nodes, Pods=pods, PodGroups=[BuildPodGroup("j", "ns", "q", 1, None, "Inqueue")],
                          Queues=[BuildQueue("q", 1, None)])
    tiers = [[PluginOption.defaults("priority"), PluginOption.defaults("gang"), PluginOption.defaults("predicates")]]
    snap = tc.RegisterSession(tiers, actions=("allocate", "preempt", "reclaim"), percentage_nodes_to_find=50,
                              min_nodes_to_find=1, last_processed_node_index=7, enable_predicate_error_cache=False)
    calls = [("c", 2, 1, 1, [1]), ("f", 1, 1, 0, [4]), ("a", 5, 2, 2, [0, 1]),  # inter-job phase
             ("c", 2, 1, 1, [1]),  # intra-job phase
             ("c", 2, 1, 0, [3]), ("f", 1, 1, 0, [4]), ("a", 5, 2, 2, [0, 1])]  # reclaim
    return snap, {"calls": calls, "index": {"preempt": 1, "reclaim": 2}, "preempt": [], "reclaim": []}


def _wide_case(mode):
    """Four 2-CPU nodes, no allocate (no NodesFitErrors entry: every task scans the NodeList), percentage 50,
    min-nodes-to-find 1: numNodesToFind(4) = 2; lastProcessedNodeIndex 3. Job "v" (priority 1) runs one preemptable
    2-CPU pod on n0 and one on n3 (v-0, v-3); n1 and n2 are empty. Job "p" (priority 10, minMember 1, Inqueue) has one
    2-CPU pending pod p-0. No scoring plugin: every node scores 0.
    PredicateNodes of p-0: start 3, n3 and n0 pass: predicateNodes [n3, n0], processed 2, index (3 + 2) % 4 = 1."""
    nodes = [BuildNode(f"n{i}", BuildResourceList("2", "4G", ("pods", "10"))) for i in range(4)]
    pods = [_pod("v-0", "n0", labels=PREEMPTABLE), _pod("v-3", "n3", labels=PREEMPTABLE), _pod("p-0", "")]
    vq, pq = ("q", "q") if mode != "reclaim" else ("qv", "qp")
    pgs = [BuildPodGroup("v", "ns", vq, 1, None, "Running"), BuildPodGroup("p", "ns", pq, 1, None, "Inqueue")]
    pgs[0].priority, pgs[1].priority = 1, 10
    queues = [BuildQueue(q, 1, None) for q in sorted({vq, pq})]
    tc = TestCommonStruct(Name=f"samp-{mode}", Nodes=nodes, Pods=pods, PodGroups=pgs, Queues=queues)
    tiers = [[PluginOption.make("priority", EnabledTaskOrder=True, EnabledJobOrder=True, EnabledPreemptable=True,
                                EnabledJobStarving=True),
              PluginOption.make("gang", EnabledJobPipelined=True, EnabledJobStarving=True),
              PluginOption.make("conformance", EnabledReclaimable=True)]]
    action = "reclaim" if mode == "reclaim" else "preempt"
    snap = tc.RegisterSession(tiers, actions=(action,), percentage_nodes_to_find=50, min_nodes_to_find=1,
                              last_processed_node_index=3, enable_predicate_error_cache=False)
    if mode == "topo":
        snap.preempt_args = PreemptArguments(topology_aware=True, min_candidate_nodes_percentage=10,
                                             min_candidate_nodes_absolute=1, max_candidate_nodes_absolute=1)
        snap.preempt_seed, snap.now_ns = 0, 0
    return snap, action


def tie_case():
    """_wide_case, preempt in its normal reading (p and v in one queue). util.PrioritizeNodes gives both predicate nodes
    0; util.SortNodes keeps the order PrioritizeNodes appended them in, scan order (scheduler_helper.go:75-140), so n3 is
    tried before n0, although n0 has the lower NodeList index. On n3 the priority plugin votes v-3 (job priority 1 < 10,
    priority.go:110-148), ValidateVictims holds (0 + 2 >= 2), v-3 is evicted and p-0 pipelined there."""
    snap, action = _wide_case("tie")
    return snap, {"calls": [("p-0", 4, 2, 1, [3, 0])], "index": {action: 1},
                  "preempt": [("evict", "v-3", 3), ("pipeline", "p-0", 3)]}


def reclaim_case():
    """_wide_case, reclaim: p in queue qp, v in queue qv (reclaimable), conformance votes v's non-critical pods
    (conformance.go:46-63). reclaimForTask walks predicateNodes as they come (reclaim.go:178-186): n3 first, where v-3
    is reclaimed and p-0 pipelined; in NodeList order n0 would have been first."""
    snap, action = _wide_case("reclaim")
    return snap, {"calls": [("p-0", 4, 2, 1, [3, 0])], "index": {action: 1},
                  "reclaim": [("evict", "v-3", 3), ("pipeline", "p-0", 3)]}


def topo_case():
    """_wide_case, preempt in its topology-aware reading, offset seed 0, numCandidates clamped to 1 (10 % of 2 nodes is
    0, minCandidateNodesAbsolute 1, maxCandidateNodesAbsolute 1; preempt.go:581-597). The first dry run (k = 0) starts at
    splitmix64(0) mod len(predicateNodes) = 16294208416658607535 mod 2 = 1, a position in predicateNodes [n3, n0]: n0.
    Its dry run succeeds with victim v-0, the one candidate, so v-0 is evicted and p-0 pipelined on n0. Positions
    counted in NodeList order ([n0, n3]) would have given n3."""
    snap, action = _wide_case("topo")
    return snap, {"calls": [("p-0", 4, 2, 1, [3, 0])], "index": {action: 1},
                  "preempt": [("evict", "v-0", 0), ("pipeline", "p-0", 0)]}


def kinds_case():
    """Allocate's NodesFitErrors entries (allocate.go:599-647, job_info.go:881-902). Two 1-CPU nodes; one job (minMember
    1, so NeedContinueAllocating holds) of 2-CPU pending pods that fit nowhere, in task order: x1, x2 (role x), y1, y2
    (role y), u1, u2, u3 (no task-spec: the empty role). x1 and y1 fail the predicate: entries with node errors; x2 and
    y2 are skipped through TaskHasFitErrors (their role has an entry): entries without node errors; TaskHasFitErrors is
    false for the empty role, so u1, u2 and u3 each fail the predicate: node errors."""
    nodes = [BuildNode(f"n{i}", BuildResourceList("1", "1G", ("pods", "10"))) for i in range(2)]
    spec = [("x1", "x"), ("x2", "x"), ("y1", "y"), ("y2", "y"), ("u1", None), ("u2", None), ("u3", None)]
    pods = [_pod(f"k-{n}", "", 70 - 10 * i, r) for i, (n, r) in enumerate(spec)]
    tc = TestCommonStruct(Name="samp-kinds", Nodes=nodes, Pods=pods, PodGroups=[BuildPodGroup("k", "ns", "q", 1, None, "Inqueue")],
                          Queues=[BuildQueue("q", 1, None)])
    tiers = [[PluginOption.defaults("priority"), PluginOption.defaults("gang"), PluginOption.defaults("predicates")]]
    snap = tc.RegisterSession(tiers, actions=("allocate", "preempt"), percentage_nodes_to_find=50, min_nodes_to_find=1,
                              enable_predicate_error_cache=False)
    return snap, {f"k-{n}": 0 if n in ("x2", "y2") else 1 for n, _ in spec}


def task_index(snap, name):
    return [k.split("/")[-1] for k in snap.task_keys].index(name)


def statements(snap, res):
    """An evicting action's committed operations as (kind, pod name, node)."""
    out = []
    for d in res.decisions:
        if int(d["kind"]) == 2:
            out.append(("evict", snap.running_task_keys[int(d["task"])].split("/")[-1], int(d["node"])))
        else:
            out.append(("pipeline", snap.task_keys[int(d["task"])].split("/")[-1], int(d["node"])))
    return out


def expected_calls(snap, calls):
    def tname(n):
        return n if "-" in n else "j-" + n
    return [{"task": task_index(snap, tname(t)), "P": P, "processed": proc, "index": idx, "nodes": nodes}
            for t, P, proc, idx, nodes in calls]


CASES = {"chain": chain_case, "tie": tie_case, "reclaim": reclaim_case, "topo": topo_case}
