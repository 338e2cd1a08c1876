"""Hand-derived sessions for reclaim with a nominated pending pod (Pod.Status.NominatedNodeName), and the random family
the H100 tests run. Reclaim never reads the nominated node: reclaimForTask checks the preemptor's PreemptionPolicy
(reclaim.go:140-143) and walks predicateNodes in NodeList order (reclaim.go:170-186); only preempt's
taskEligibleToPreempt (preempt.go:436-470) reads NominatedNodeName."""
from __future__ import annotations

import random

from volcano_b200.api import BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct


def reclaim_case(nominated="n0", actions=("reclaim",)):
    """Two 2-CPU nodes. n0 runs w-0 (job w, queue qp, preemptable); n1 runs v-1 (job v, queue qv, preemptable). The
    reclaimer p-0 (job p, queue qp, minMember 1, Inqueue) requests 2 CPUs and is nominated to `nominated` (n0, or a name
    not in the session). reclaim, node n0 first: the filter keeps Running tasks of other, reclaimable queues
    (reclaim.go:184-199), and w-0 sits in p's own queue, so n0 has no candidate. n1: conformance votes v-1 (not
    critical, conformance.go:46-63); ValidateVictims holds (0 + 2 >= 2); v-1 is evicted and p-0 pipelined on n1. The
    nomination to n0 plays no part."""
    nodes = [BuildNode(f"n{i}", BuildResourceList("2", "4G", ("pods", "10"))) for i in range(2)]
    lab = {"volcano.sh/preemptable": "true"}
    pods = [BuildPod("ns", "w-0", "n0", "Running", BuildResourceList("2", "1G"), "w", lab),
            BuildPod("ns", "v-1", "n1", "Running", BuildResourceList("2", "1G"), "v", lab),
            BuildPod("ns", "p-0", "", "Pending", BuildResourceList("2", "1G"), "p", {})]
    pods[2].nominated_node_name = nominated
    pgs = [BuildPodGroup("w", "ns", "qp", 1, None, "Running"), BuildPodGroup("v", "ns", "qv", 1, None, "Running"),
           BuildPodGroup("p", "ns", "qp", 1, None, "Inqueue")]
    tc = TestCommonStruct(Name="nominated-reclaim", Nodes=nodes, Pods=pods, PodGroups=pgs,
                          Queues=[BuildQueue("qp", 1, None), BuildQueue("qv", 1, None)])
    tiers = [[PluginOption.make("priority", EnabledTaskOrder=True, EnabledJobOrder=True, EnabledJobStarving=True),
              PluginOption.make("gang", EnabledJobPipelined=True, EnabledJobStarving=True),
              PluginOption.make("conformance", EnabledReclaimable=True)]]
    snap = tc.RegisterSession(tiers, actions=actions)
    return snap, [("evict", "v-1", 1), ("pipeline", "p-0", 1)]


def nominate(tc, seed):
    """make_case's cluster with NominatedNodeName on about half the pending pods: a node of the session, or a name that
    is not one. Returns how many pods carry a name."""
    rnd = random.Random(seed * 7727 + 1)
    n = 0
    for p in tc.Pods:
        if not p.node_name and rnd.random() < 0.5:
            p.nominated_node_name = rnd.choice([nd.name for nd in tc.Nodes] + ["gone"])
            n += 1
    return n
