"""Hand-derived sessions for preempt's normal reading with PreferNoSchedule taints. Each builder returns the snapshot and
the statements of preempt as (kind, pod name, node), derived in its docstring from the reference:

- util.PrioritizeNodes (scheduler_helper.go:76-136) sums, per node of predicateNodes, the NodeOrderFn total and the
  BatchNodeOrderFn entries. nodeorder's BatchNodeOrderFn (nodeorder.go:332-384) scores TaintToleration: the count of
  PreferNoSchedule taints the pod does not tolerate, normalised by DefaultNormalizeScore(MaxNodeScore, reverse) over the
  nodes it was given: 100 - 100 * count / max in int64 (100 for every node when max is 0), times tainttoleration.weight.
- predicateNodes is every node passing PredicateForPreemptAction without sampling, and the sampled list under it
  (preempt.go:293-325), in scan order; util.SortNodes keeps that order among equal scores.
- Here only two scorers are on: nodeaffinity (weight 2, the raw sum of matching preferred weights, nodeorder.go:314-330)
  and TaintToleration (weight 3); the other nodeorder weights are 0.

Node names n0.. are NodeList positions. Every node has 2 CPUs and runs at most one 2-CPU pod; v-* pods (job v, priority
1) are preemptable, w-* pods (job w) are not, so a node running a w pod is a predicate node but never a candidate. The
preemptor p-0 (job p, priority 10, minMember 1) requests 2 CPUs; priority votes v's pods (priority.go:110-148)."""
from __future__ import annotations

from volcano_b200.api import (BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList, NodeSelectorRequirement,
                              Taint, Toleration)
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct

NODEORDER_ARGS = {"leastrequested.weight": 0, "mostrequested.weight": 0, "balancedresource.weight": 0,
                  "nodeaffinity.weight": 2, "tainttoleration.weight": 3}


def _session(layout, tolerate=(), **conf):
    """layout: per node (running pod prefix "v" / "w" / None, soft-taint count, preferred by the preemptor)."""
    nodes, pods = [], []
    for i, (run, n_soft, fav) in enumerate(layout):
        node = BuildNode(f"n{i}", BuildResourceList("2", "4G", ("pods", "10")), {"fav": "y"} if fav else {})
        node.taints = [Taint(f"t{k}", "", "PreferNoSchedule") for k in range(n_soft)]
        nodes.append(node)
        if run:
            lab = {"volcano.sh/preemptable": "true" if run == "v" else "false"}
            pods.append(BuildPod("ns", f"{run}-{i}", f"n{i}", "Running", BuildResourceList("2", "1G"), run, lab))
    p = BuildPod("ns", "p-0", "", "Pending", BuildResourceList("2", "1G"), "p", {})
    p.affinity_preferred = [(100, [NodeSelectorRequirement("fav", "In", ("y",))])]
    p.tolerations = [Toleration(k, "Exists", "", "PreferNoSchedule") for k in tolerate]
    pods.append(p)
    pgs = [BuildPodGroup("v", "ns", "q", 1, None, "Running"), BuildPodGroup("w", "ns", "q", 1, None, "Running"),
           BuildPodGroup("p", "ns", "q", 1, None, "Inqueue")]
    pgs[0].priority, pgs[1].priority, pgs[2].priority = 1, 1, 10
    tc = TestCommonStruct(Name="soft", Nodes=nodes, Pods=pods, PodGroups=pgs, Queues=[BuildQueue("q", 1, None)])
    tiers = [[PluginOption.make("priority", EnabledTaskOrder=True, EnabledJobOrder=True, EnabledPreemptable=True,
                                EnabledJobStarving=True),
              PluginOption.make("gang", EnabledJobPipelined=True, EnabledJobStarving=True),
              PluginOption.make("nodeorder", NODEORDER_ARGS, EnabledNodeOrder=True)]]
    return tc.RegisterSession(tiers, actions=("preempt",), **conf)


# n0: v pod, 1 soft taint, preferred (order 200); n1: v pod; n2: w pod, 3 soft taints; n3: w pod
_MAX_LAYOUT = [("v", 1, True), ("v", 0, False), ("w", 3, False), ("w", 0, False)]


def all_nodes_case():
    """_MAX_LAYOUT without sampling. predicateNodes are n0..n3 and the maximum count is 3, on n2, which is not a
    candidate (w-2 is not preemptable and n2 has no FutureIdle). Scores: n0 200 + 3 * (100 - 100 * 1 / 3) = 200 + 3 * 67
    = 401; n1 0 + 3 * 100 = 300; n2 3 * 0 = 0; n3 300. n0 is tried first: v-0 is evicted and p-0 pipelined there. A
    maximum taken over the candidates n0, n1 alone (1) would give n0 200 and n1 300, and n1 would win."""
    snap = _session(_MAX_LAYOUT)
    return snap, [("evict", "v-0", 0), ("pipeline", "p-0", 0)]


def sample_case():
    """_MAX_LAYOUT under sampling: percentage 50, min-nodes-to-find 1, lastProcessedNodeIndex 0. numNodesToFind(4) = 2
    (scheduler_helper.go:54-73); the scan from 0 keeps n0, n1: predicateNodes [n0, n1], and the maximum over them is 1.
    Scores: n0 200 + 3 * (100 - 100) = 200; n1 300. n1 is tried first: v-1 is evicted and p-0 pipelined there, where
    the maximum over every predicate node (3, on n2 outside the sample) chose n0."""
    snap = _session(_MAX_LAYOUT, percentage_nodes_to_find=50, min_nodes_to_find=1, last_processed_node_index=0,
                    enable_predicate_error_cache=False)
    return snap, [("evict", "v-1", 1), ("pipeline", "p-0", 1)]


def truncation_case():
    """n0: v pod, no taint; n1: w pod, no taint; n2: v pod, 1 soft taint; n3: w pod, 150 soft taints. No preferred
    node. Sampling: percentage 75, min-nodes-to-find 1, lastProcessedNodeIndex 2: numNodesToFind(4) = 3, and the scan
    from 2 keeps n2, n3, n0 in that order. The maximum is 150. Scores: n2 3 * (100 - 100 * 1 / 150) = 3 * (100 - 0) =
    300 (int64 division truncates); n0 300; n3 3 * (100 - 100) = 0. n2 and n0 tie; SortNodes keeps scan order, so n2 is
    tried first: v-2 is evicted and p-0 pipelined on n2 (NodeList order would have given n0)."""
    snap = _session([("v", 0, False), ("w", 0, False), ("v", 1, False), ("w", 150, False)], percentage_nodes_to_find=75,
                    min_nodes_to_find=1, last_processed_node_index=2, enable_predicate_error_cache=False)
    return snap, [("evict", "v-2", 2), ("pipeline", "p-0", 2)]


def zero_max_case():
    """n0: v pod, no taint; n1: v pod, preferred (order 200), one soft taint t0, which p-0 tolerates (effect
    PreferNoSchedule, operator Exists). The session still carries a PreferNoSchedule taint, but p-0's counts are 0 on
    every node, so the maximum is 0 and every node gets 3 * 100 = 300: n0 300, n1 500. n1 is tried first: v-1 is
    evicted and p-0 pipelined there. Were t0 not tolerated, the maximum would be 1, n1 would score 200 and n0 would
    win."""
    snap = _session([("v", 0, False), ("v", 1, True)], tolerate=("t0",))
    return snap, [("evict", "v-1", 1), ("pipeline", "p-0", 1)]


CASES = {"all_nodes": all_nodes_case, "sample": sample_case, "truncation": truncation_case, "zero_max": zero_max_case}
