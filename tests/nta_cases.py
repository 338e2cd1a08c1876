"""Hand-derived preempt and reclaim sessions with the network-topology-aware plugin. CASES[name]() -> (snapshot, sorted
evicted pod keys).

The cluster of every case: four nodes of 8 cpus and 32G, n0 and n2 in HyperNode hnA, n1 and n3 in hnB (tier 1; the
cluster top hypernode is tier 2 and holds every node). Each node runs one pod of job "low" (priority 1, minMember 0):
6 cpus and 2G on hnA's nodes, 6 cpus and 16G on hnB's. A preemptor of 4 cpus fits no node without an eviction. The
plugin's defaults: weight 1, cpu and memory weight 1, fading 0.8, binpacking of normal pods on.

hyperNodeResourceCache at open: hnA used (12 cpus, 4G), hnB used (12 cpus, 32G), each of (16 cpus, 64G). For a pod of
4 cpus and 1G, getPodHyperNodeBinPackingScore (network_topology_aware.go:500-539) gives hnA (16/16 + 5/64) / 2 =
0.5390625 and hnB (16/16 + 33/64) / 2 = 0.7578125; the tier-2 term is the same on every node. util.SortNodes then walks
n1, n3 (hnB), n0, n2 (hnA); without the plugin every score is 0 and the walk is n0, n1, n2, n3."""
from __future__ import annotations

from volcano_b200.api import (BuildHyperNode, BuildNode, BuildPod, BuildPodGroupWithNetWorkTopologies, BuildPodGroupWithPrio,
                              BuildQueue, BuildResourceList)
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct


def _job(name, queue, min_member, prio, soft=False, phase="Inqueue"):
    if soft:
        pg = BuildPodGroupWithNetWorkTopologies(name, "ns", "", queue, min_member, None, phase, "soft", 0)
        pg.priority = prio
        return pg
    return BuildPodGroupWithPrio(name, "ns", queue, min_member, None, phase, prio)


def _pending(job, n, cpu="4", mem="1G"):
    return [BuildPod("ns", f"{job}-{i}", "", "Pending", BuildResourceList(cpu, mem), job) for i in range(n)]


def _session(pending_jobs, pending_pods, actions, nta=True, low_soft=False, tdm=False):
    tc = TestCommonStruct(Name="nta")
    tc.Nodes = [BuildNode(f"n{i}", BuildResourceList("8", "32G", ("pods", "10"))) for i in range(4)]
    tc.HyperNodes = [BuildHyperNode("hnA", 1, [("n0", "Node"), ("n2", "Node")]),
                     BuildHyperNode("hnB", 1, [("n1", "Node"), ("n3", "Node")])]
    tc.Queues = [BuildQueue("q", 1), BuildQueue("qp", 1)]
    tc.PodGroups = [_job("low", "q", 0, 1, soft=low_soft, phase="Running")] + list(pending_jobs)
    tc.Pods = [BuildPod("ns", f"r{i}", f"n{i}", "Running", BuildResourceList("6", "2G" if i % 2 == 0 else "16G"), "low")
               for i in range(4)] + list(pending_pods)
    tiers = [[PluginOption.defaults(n) for n in ("priority", "gang", "conformance")]]
    if nta:
        tiers.append([PluginOption.defaults("network-topology-aware")])
    if tdm:
        tiers[-1].append(PluginOption.defaults("tdm"))
    return tc.RegisterSession(tiers, actions=actions)


def term_changes_the_node(nta=True):
    """Job "high" (queue q, priority 10, one pod of 4 cpus / 1G). SortNodes walks n1 first (hnB scores 0.7578125 against
    hnA's 0.5390625); r1 (priority 1) is the victim and frees 6 cpus: r1 is evicted. Without the plugin n0 comes first
    and r0 is evicted."""
    return _session([_job("high", "q", 1, 10)], _pending("high", 1), ("preempt",), nta=nta), (["ns/r1"] if nta else ["ns/r0"])


def topology_job_skipped_and_evicted():
    """Job "low" has a soft network topology, and so has pending job "topo" (priority 10). Pending job "high" (priority 5)
    has none. preempt.go:132-137 leaves "topo" out of the preemptors, so only "high" preempts: n1 first, r1 (a pod of a
    topology job, priority 1) is its victim and is evicted, and high's pod is pipelined there."""
    jobs = [_job("topo", "q", 1, 10, soft=True), _job("high", "q", 1, 5)]
    return _session(jobs, _pending("topo", 1) + _pending("high", 1), ("preempt",), low_soft=True), ["ns/r1"]


def topology_job_reclaims():
    """Job "rc" (queue qp, soft network topology, one pod of 4 cpus / 1G) reclaims: reclaim.go has no topology skip. The
    walk is NodeList order, n0 first; conformance and gang return r0 (low's minMember is 0), which is evicted."""
    return _session([_job("rc", "qp", 1, 1, soft=True)], _pending("rc", 1), ("reclaim",)), ["ns/r0"]


def discard_restores_used():
    """Job "big" (priority 10, minMember 9, nine pods of 4 cpus / 1G), then job "small" (priority 5, one such pod). An
    evicted 6-cpu pod leaves room for two of big's pods on its node (ValidateVictims accepts an empty victim list when
    FutureIdle already fits, scheduler_helper.go:313-329), so big's pods fill the four nodes two by two and the ninth
    finds no room. big is not pipelined (gang: 8 < 9) and its statement is discarded: Discard runs the DeallocateFunc
    of each pipelined pod and the AllocateFunc of each unevicted one, so hyperNodeResourceCache is back at its opening
    values. small then walks n1 first again and evicts r1. Had the discard left the cache where the eight placements put
    it (16 cpus used on both hypernodes: both score 0 on the tier), the scores would tie and n0 would come first."""
    jobs = [_job("big", "q", 9, 10), _job("small", "q", 1, 5)]
    return _session(jobs, _pending("big", 9) + _pending("small", 1), ("preempt",)), ["ns/r1"]


def reclaim_then_preempt():
    """Actions reclaim, then preempt. Reclaim: job "rc" (queue qp, soft topology, one pod of 6 cpus / 31G) takes n0 (first
    in NodeList order): r0 is evicted and rc's pod pipelined there, so hnA's used becomes (12 - 6 + 6, 4 - 2 + 31) =
    (12 cpus, 33G). Job "high" (queue q) gets nothing from reclaim (no running pod of another queue). Preempt: high's pod
    (4 cpus / 1G) scores hnA (16/16 + 34/64) / 2 = 0.765625 and hnB 0.7578125, so the walk is n0, n2, n1, n3; n0 is no
    candidate (FutureIdle 2 + 6 - 6 = 2 cpus, no victim left), n2 is: r2 is evicted. Read at its opening values the
    cache would have sent high to n1."""
    jobs = [_job("rc", "qp", 1, 1, soft=True), _job("high", "q", 1, 10)]
    return _session(jobs, _pending("rc", 1, cpu="6", mem="31G") + _pending("high", 1), ("reclaim", "preempt")), ["ns/r0", "ns/r2"]


def with_tdm():
    """term_changes_the_node's session with the tdm plugin beside network-topology-aware: preempt and reclaim refuse it."""
    return _session([_job("high", "q", 1, 10)], _pending("high", 1), ("preempt",), tdm=True)


CASES = {f.__name__: f for f in (term_changes_the_node, topology_job_skipped_and_evicted, topology_job_reclaims,
                                 discard_restores_used, reclaim_then_preempt)}
