"""Hand-derived preempt and reclaim sessions with the pdb and cdp plugins. Each case's docstring derives its evictions
from the Go code (plugins/pdb/pdb.go:65-126, plugins/cdp/cdp.go:56-110, framework/session_plugins.go:211-307).
CASES[name]() -> (snapshot, sorted evicted pod keys)."""
from __future__ import annotations

from volcano_b200.api import BuildNode, BuildPDB, BuildPod, BuildPodGroupWithPrio, BuildQueue, BuildResourceList
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct

NOW = 10 ** 18  # SchedulerConf.now_ns: time.Now() of the session
S = 10 ** 9


def _running(name, node, labels=None, group="low", cpu="1", **kw):
    p = BuildPod("ns", name, node, "Running", BuildResourceList(cpu, "1G"), group, labels or {})
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _session(nodes, running, pdbs, tiers, preemptor_cpu="1", n_preemptors=1, actions=("preempt",), reclaim=False):
    """Nodes of `nodes` cpus each, full with `running` (job "low", priority 1, queue q); preemptors of job "high"
    (priority 10): in queue q for preempt, in queue qp for reclaim (q then reclaimable)."""
    tc = TestCommonStruct(Name="guard")
    tc.Nodes = [BuildNode(f"n{i}", BuildResourceList(str(c), "16G", ("pods", "10"))) for i, c in enumerate(nodes)]
    tc.Queues = [BuildQueue("q", 1), BuildQueue("qp", 1)]
    tc.PodGroups = [BuildPodGroupWithPrio("low", "ns", "q", 1, None, "Running", 1),
                    BuildPodGroupWithPrio("high", "ns", "qp" if reclaim else "q", n_preemptors, None, "Inqueue", 10)]
    tc.Pods = list(running) + [BuildPod("ns", f"p-{i}", "", "Pending", BuildResourceList(preemptor_cpu, "1G"), "high")
                               for i in range(n_preemptors)]
    tc.PDBs = list(pdbs)
    return tc.RegisterSession(tiers, actions=actions, now_ns=NOW)


def _tiers(*tiers):
    return [[PluginOption.defaults(n) for n in t] for t in tiers]


def budget_one_two_pods():
    """One PDB app=a with DisruptionsAllowed 1 over r-0 and r-1 on n0 (2 cpus, full). Preemptor p-0 (1 cpu, job priority 10
    over 1). Tier [priority, pdb]: priority returns both; pdb walks r-0 (budget 1 -> 0, a victim), then r-1 (0 -> -1,
    violated, kept) and returns [r-0]. The intersection is [r-0]; ValidateVictims 0 + 1 >= 1 holds; r-0 is evicted."""
    run = [_running("r-0", "n0", {"app": "a"}), _running("r-1", "n0", {"app": "a"})]
    return _session([2], run, [BuildPDB("ns", "pdb", {"app": "a"}, 1)], _tiers(["priority", "pdb"])), ["ns/r-0"]


def budget_one_needs_two():
    """As budget_one_two_pods, but p-0 requests 2 cpus: the victims are still [r-0] (r-1 is protected), ValidateVictims
    0 + 1 >= 2 fails on the only node, nothing is evicted."""
    run = [_running("r-0", "n0", {"app": "a"}), _running("r-1", "n0", {"app": "a"})]
    return _session([2], run, [BuildPDB("ns", "pdb", {"app": "a"}, 1)], _tiers(["priority", "pdb"]), preemptor_cpu="2"), []


def overlapping_pdbs():
    """r-0 {app: a, tier: x}, r-1 {app: a} on n0. PDB a (app=a) allows 2, PDB x (tier=x) allows 0. r-0: a 2 -> 1, x 0 -> -1:
    kept. r-1: a 1 -> 0: a victim. p-0 (1 cpu) evicts r-1."""
    run = [_running("r-0", "n0", {"app": "a", "tier": "x"}), _running("r-1", "n0", {"app": "a"})]
    pdbs = [BuildPDB("ns", "a", {"app": "a"}, 2), BuildPDB("ns", "x", {"tier": "x"}, 0)]
    return _session([2], run, pdbs, _tiers(["priority", "pdb"])), ["ns/r-1"]


def disrupted_pod():
    """PDB app=a allows 0 but lists r-0 in DisruptedPods: r-0 is not counted (pdb.go:105-109) and is a victim; r-1 is
    counted (0 -> -1) and kept. p-0 evicts r-0."""
    run = [_running("r-0", "n0", {"app": "a"}), _running("r-1", "n0", {"app": "a"})]
    return _session([2], run, [BuildPDB("ns", "pdb", {"app": "a"}, 0, ["r-0"])], _tiers(["priority", "pdb"])), ["ns/r-0"]


def unlabeled_pod():
    """r-0 has no labels: pdb skips it (pdb.go:87-90) and returns nothing, with no PDB at all. The tier [priority, pdb]
    is voided, no other tier: no victim, nothing is evicted."""
    return _session([1], [_running("r-0", "n0")], [], _tiers(["priority", "pdb"])), []


def per_call_reset():
    """Two 1-cpu nodes, r-0 on n0 and r-1 on n1, PDB app=a allows 1; job high has two 1-cpu preemptors. Each
    ssn.Preemptable call sees one node's pods and starts from DisruptionsAllowed again (pdb.go:75-79): p-0 evicts r-0 on
    n0, p-1 evicts r-1 on n1. Two evictions under a budget of one, as the reference does."""
    run = [_running("r-0", "n0", {"app": "a"}), _running("r-1", "n1", {"app": "a"})]
    return (_session([1, 1], run, [BuildPDB("ns", "pdb", {"app": "a"}, 1)], _tiers(["priority", "pdb"]), n_preemptors=2),
            ["ns/r-0", "ns/r-1"])


def pdb_last_voter_nil_reset():
    """Tiers [priority, pdb] then [conformance]. pdb returns nothing (r-0 counted by a PDB allowing 0), so the first tier is
    voided (victims = nil, session_plugins.go:232-235) and conformance decides: r-0 is not critical and is evicted."""
    run = [_running("r-0", "n0", {"app": "a"})]
    return (_session([1], run, [BuildPDB("ns", "pdb", {"app": "a"}, 0)], _tiers(["priority", "pdb"], ["conformance"])),
            ["ns/r-0"])


def cdp_until_now():
    """r-0 scheduled 100 s before now with a 100s cooldown: LastTransitionTime + cooldown == now, and Time.After is strict,
    so cdp returns it; r-1 scheduled 99 s before now is kept. Preemptor p-0 (1 cpu) evicts r-0."""
    run = [_running("r-0", "n0", {"volcano.sh/cooldown-time": "100s"}, scheduled_time=NOW - 100 * S),
           _running("r-1", "n0", annotations={"volcano.sh/cooldown-time": "100s"}, scheduled_time=NOW - 99 * S)]
    return _session([2], run, [], _tiers(["priority", "cdp"])), ["ns/r-0"]


def reclaim_both():
    """Reclaim: p-0 (queue qp, 1 cpu) against n0 (3 cpus) full with r-0, r-1, r-2 of queue q. Tiers [priority] (JobStarving
    only: it registers no ReclaimableFn) then [pdb, cdp]. pdb: r-0 counted by a PDB allowing 0 -> kept; cdp: r-1 in
    cooldown (1h from 10 s ago) -> kept; r-2 passes both. The victims are [r-2], which is evicted."""
    run = [_running("r-0", "n0", {"app": "a"}), _running("r-1", "n0", {"volcano.sh/cooldown-time": "1h"}, scheduled_time=NOW - 10 * S),
           _running("r-2", "n0", {"app": "b"})]
    return (_session([3], run, [BuildPDB("ns", "pdb", {"app": "a"}, 0)], _tiers(["priority"], ["pdb", "cdp"]),
                     actions=("reclaim",), reclaim=True), ["ns/r-2"])


CASES = {f.__name__: f for f in (budget_one_two_pods, budget_one_needs_two, overlapping_pdbs, disrupted_pod, unlabeled_pod,
                                 per_call_reset, pdb_last_voter_nil_reset, cdp_until_now, reclaim_both)}
