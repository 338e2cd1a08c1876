"""Random API-level clusters for the preempt and reclaim actions: nodes filled with running pods of several jobs and
queues (preemptable / not, task and job priorities, critical pods, Bound pods), starving jobs with pending pods, queue
capabilities / priorities / closed and non-reclaimable queues, random subsets and tier splits of the plugins that vote
on victims (conformance, gang, priority, drf, proportion) plus the scoring plugins, and a random action list out of
allocate / preempt / reclaim.  make_case(seed) -> (TestCommonStruct, tiers, actions); used by tests/test_gpu_fuzz.py and
`python tools/fuzz_evict.py <first> <last>` on a GPU box (CUDA path vs CPU oracle, statement by statement)."""
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from volcano_b200.api import (BuildNode, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList)  # noqa: E402
from volcano_b200.snapshot import PluginOption  # noqa: E402
from volcano_b200.uthelper import TestCommonStruct  # noqa: E402


def make_case(seed):
    rnd = random.Random(seed * 104729 + 7)
    n_nodes = rnd.randint(1, 6)
    nodes = []
    for i in range(n_nodes):
        labels = {"zone": rnd.choice(["a", "b"])} if rnd.random() < 0.4 else {}
        nodes.append(BuildNode(f"n{i}", BuildResourceList(str(rnd.choice([2, 3, 4])), rnd.choice(["4G", "8G", "16G"]),
                                                          ("pods", str(rnd.choice([3, 6, 20])))), labels))
    n_queues = rnd.randint(1, 3)
    queues = []
    for q in range(n_queues):
        cap = BuildResourceList(str(rnd.choice([2, 4, 8, 16])), rnd.choice(["4G", "8G", "32G"])) if rnd.random() < 0.4 else None
        qu = BuildQueue(f"q{q}", rnd.randint(1, 4), cap)
        qu.priority = rnd.choice([0, 0, 1, 5])
        if rnd.random() < 0.1:
            qu.state = "Closed"
        if rnd.random() < 0.15:
            qu.reclaimable = False
        queues.append(qu)
    pgs, pods = [], []
    n_jobs = rnd.randint(2, 7)
    for j in range(n_jobs):
        q = rnd.randrange(n_queues)
        n_run, n_pend = rnd.randint(0, 5), rnd.randint(0, 4)
        size = n_run + n_pend
        if size == 0:
            n_pend = size = 1
        min_member = rnd.choice([0, 1, max(1, size // 2), size, size + 1])
        roles = rnd.random() < 0.3
        tmm = None
        if roles and rnd.random() < 0.5:
            tmm = {"w": rnd.randint(0, max(1, size // 2))}
        phase = rnd.choice(["Inqueue", "Running", "Running", "Pending"])
        pg = BuildPodGroup(f"pg{j}", "ns", f"q{q}", min_member, tmm, phase)
        pg.priority = rnd.choice([0, 10, 10, 1000])
        pgs.append(pg)
        req = BuildResourceList(rnd.choice(["500m", "1", "2", "3"]), rnd.choice(["1G", "2G", "4G"]))
        sel = {"zone": rnd.choice(["a", "b"])} if rnd.random() < 0.15 else {}
        for k in range(size):
            running = k < n_run
            role = ("m" if k == 0 else "w") if roles else "w"
            labels = {"volcano.sh/task-spec": role}
            r = rnd.random()
            if r < 0.35:
                labels["volcano.sh/preemptable"] = "true"
            elif r < 0.55:
                labels["volcano.sh/preemptable"] = "false"
            p = BuildPod("ns" if rnd.random() > 0.05 else "kube-system", f"j{j}-{role}-{k}", rnd.choice(nodes).name if running else "",
                         "Running" if running and rnd.random() > 0.1 else "Pending", req, f"pg{j}", labels, {} if running else sel)
            if p.namespace != "ns":
                p.group_name = f"pg{j}"
            if rnd.random() < 0.3:
                p.priority = rnd.choice([1, 5, 100])
            if not running and rnd.random() < 0.08:
                p.preemption_policy = "Never"
            if running and rnd.random() < 0.05:
                p.priority_class_name = "system-node-critical"
            p.creation_ts = rnd.randint(0, 3)
            pods.append(p)
    # pods of a kube-system namespace belong to a job id of their own namespace: keep them in "ns" groups only
    for p in pods:
        if p.namespace != "ns":
            p.namespace = "ns"
            p.priority_class_name = "system-cluster-critical"
            p.uid = ""
            p.__post_init__()
    tiers, actions = _plugins_and_actions(rnd)
    tc = TestCommonStruct(Name=f"evict-fuzz{seed}", Nodes=nodes, Pods=pods, PodGroups=pgs, Queues=queues)
    return tc, tiers, actions


def make_wide_case(seed):
    """Wide clusters: 40-3 000 mostly identical nodes (equal scores: ties across every warp of the pick kernel, and idle
    nodes that pass the node filter but offer no victim, so a preemptor walks past many candidates), a few nodes running
    more than 16 pods, and 9 or more resource names (R > 8)."""
    rnd = random.Random(seed * 7919 + 11)
    n_nodes = rnd.randint(40, 3000)
    scalars = [f"example.com/s{i}" for i in range(rnd.randint(7, 9))]
    base = BuildResourceList("16", "32G", ("pods", "110"), *[(s, "4") for s in scalars])
    odd = BuildResourceList("8", "32G", ("pods", "110"), *[(s, "4") for s in scalars])
    nodes = [BuildNode(f"n{i:04d}", odd if rnd.random() < 0.05 else base) for i in range(n_nodes)]
    queues = [BuildQueue(f"q{q}", rnd.randint(1, 4), None) for q in range(rnd.randint(2, 3))]
    # hot nodes: more than 16 running pods each, anywhere in the node list (often near its end)
    hot = sorted({rnd.choice([rnd.randrange(n_nodes), n_nodes - 1 - rnd.randrange(min(n_nodes, 64))])
                  for _ in range(rnd.randint(1, 3))})
    pgs, pods = [], []
    small = BuildResourceList("500m", "512M", *[(s, "0") for s in scalars[:2]])
    for j, node in enumerate(hot):  # one running job per hot node, 24-30 pods: 1-4 of its 16 cores left
        q = rnd.randrange(len(queues))
        n_run = rnd.randint(24, 30)
        pgs.append(BuildPodGroup(f"hot{j}", "ns", f"q{q}", rnd.choice([1, n_run // 2, n_run]), None, "Running"))
        pgs[-1].priority = rnd.choice([0, 10])
        for k in range(n_run):
            labels = {"volcano.sh/preemptable": "true"} if rnd.random() < 0.8 else {}
            pods.append(BuildPod("ns", f"hot{j}-{k}", nodes[node].name, "Running", small, f"hot{j}", labels))
    n_spread = rnd.randint(0, min(300, n_nodes))  # single running pods on random nodes
    if n_spread:
        q = rnd.randrange(len(queues))
        pgs.append(BuildPodGroup("spread", "ns", f"q{q}", 1, None, "Running"))
        for k in range(n_spread):
            pods.append(BuildPod("ns", f"spread-{k}", rnd.choice(nodes).name, "Running",
                                 BuildResourceList("2", "2G", (rnd.choice(scalars), "1")), "spread", {}))
    for j in range(rnd.randint(1, 3)):  # starving jobs: their pods need the whole of some scalar a hot node holds
        q = rnd.randrange(len(queues))
        n_pend = rnd.randint(1, 4)
        pgs.append(BuildPodGroup(f"pend{j}", "ns", f"q{q}", n_pend, None, rnd.choice(["Inqueue", "Running"])))
        pgs[-1].priority = rnd.choice([10, 1000])
        req = BuildResourceList(rnd.choice(["4", "15"]), "4G", *[(s, "1") for s in rnd.sample(scalars, rnd.randint(1, 4))])
        for k in range(n_pend):
            pods.append(BuildPod("ns", f"pend{j}-{k}", "", "Pending", req, f"pend{j}", {}))
    tiers, actions = _plugins_and_actions(rnd)
    tc = TestCommonStruct(Name=f"evict-wide{seed}", Nodes=nodes, Pods=pods, PodGroups=pgs, Queues=queues)
    return tc, tiers, tuple(a for a in actions if a != "allocate") or ("preempt",)  # allocate would fill the idle nodes


def make_topo_case(seed):
    """Topology-aware preemption: make_case's clusters with pod priorities and start times (some unset, many equal), pods
    with and without an index in their names mixed in one job (the victim order then is not a strict weak order),
    proportion with or without EnabledPredicate, and random candidate-count arguments, offset seeds and clocks.
    -> (TestCommonStruct, tiers, actions, conf keyword arguments of RegisterSession)."""
    from volcano_b200 import abi
    tc, tiers, actions = make_case(seed)
    rnd = random.Random(seed * 31337 + 5)
    for p in tc.Pods:
        if p.node_name and rnd.random() < 0.7:
            p.start_time = rnd.choice([1, 2, 3]) * 10 ** 9
        if p.node_name and rnd.random() < 0.3:  # no pod index: util.LessFn falls back to creation time for this pod
            p.name += "x"
        if p.node_name and p.priority is None and rnd.random() < 0.2:
            p.annotations["volcano.sh/task-priority"] = str(rnd.choice([2, 50]))  # TaskInfo.Priority only
    for tier in tiers:
        for opt in tier:
            if opt.name == "proportion" and rnd.random() < 0.3:
                opt.enabled &= ~abi.VC_EN_PREDICATE
    if "preempt" not in actions:
        actions = actions + ("preempt",)
    args = {"enableTopologyAwarePreemption": True, "topologyAwarePreemptWorkerNum": rnd.choice([1, 16]),
            "minCandidateNodesPercentage": rnd.choice([0, 10, 50, 100]), "minCandidateNodesAbsolute": rnd.choice([0, 1, 2, 3]),
            "maxCandidateNodesAbsolute": rnd.choice([1, 2, 100])}
    conf = {"configurations": {"preempt": args}, "preempt_seed": rnd.getrandbits(64), "now_ns": rnd.randint(0, 4) * 10 ** 9}
    return tc, tiers, actions, conf


def make_samp_case(seed):
    """Feasible-node sampling: make_case's clusters widened to 3-40 nodes (zone labels and selectors make the static
    verdicts, and so the filtered lists of starving tasks, differ from task to task), percentage-nodes-to-find 34 / 50 /
    67 with min-nodes-to-find 1, a carried lastProcessedNodeIndex anywhere in [0, 2N], allocate first in most action
    lists, and the topology-aware reading in a third of the cases. The predicate error cache is off (with it on, sessions
    whose named roles span several groups are refused). -> (TestCommonStruct, tiers, actions, conf keyword arguments)."""
    from volcano_b200.api import BuildNode, BuildResourceList
    rnd = random.Random(seed * 15485863 + 3)
    topo = rnd.random() < 0.33
    tc, tiers, actions, conf = make_topo_case(seed) if topo else (*make_case(seed), {})
    for i in range(len(tc.Nodes), rnd.randint(max(3, len(tc.Nodes)), 40)):
        labels = {"zone": rnd.choice(["a", "b"])} if rnd.random() < 0.6 else {}
        tc.Nodes.append(BuildNode(f"n{i}", BuildResourceList(str(rnd.choice([1, 2, 3, 4])), rnd.choice(["4G", "8G", "16G"]),
                                                               ("pods", str(rnd.choice([3, 6, 20])))), labels))
    if rnd.random() < 0.8 and "allocate" not in actions:
        actions = ("allocate",) + tuple(a for a in actions if a != "enqueue")
    conf.update(percentage_nodes_to_find=rnd.choice([34, 50, 67]), min_nodes_to_find=1,
                last_processed_node_index=rnd.randint(0, 2 * len(tc.Nodes)), enable_predicate_error_cache=False)
    return tc, tiers, actions, conf


def make_soft_case(seed):
    """PreferNoSchedule taints: make_case's clusters widened to 3-40 nodes, random PreferNoSchedule and NoSchedule taints
    on the nodes and tolerations (either effect, or every effect) on the pods, nodeorder always on with
    tainttoleration.weight 0 or 3 (the other scorers as make_case draws them), feasible-node sampling in half the cases
    and the topology-aware reading in a third. -> (TestCommonStruct, tiers, actions, conf keyword arguments)."""
    from volcano_b200.api import Taint, Toleration
    rnd = random.Random(seed * 2750159 + 13)
    topo = rnd.random() < 0.33
    tc, tiers, actions, conf = make_topo_case(seed) if topo else (*make_case(seed), {})
    for i in range(len(tc.Nodes), rnd.randint(max(3, len(tc.Nodes)), 40)):
        labels = {"zone": rnd.choice(["a", "b"])} if rnd.random() < 0.4 else {}
        tc.Nodes.append(BuildNode(f"n{i}", BuildResourceList(str(rnd.choice([1, 2, 3, 4])), rnd.choice(["4G", "8G", "16G"]),
                                                               ("pods", str(rnd.choice([3, 6, 20])))), labels))
    keys = ["s0", "s1", "s2", "s3"]
    for n in tc.Nodes:
        n.taints = [Taint(k, "", "PreferNoSchedule") for k in keys if rnd.random() < 0.3]
        if rnd.random() < 0.1:
            n.taints.append(Taint("h0", "", "NoSchedule"))
    for p in tc.Pods:
        if not p.node_name and rnd.random() < 0.4:
            p.tolerations = [Toleration(rnd.choice(keys + ["h0"]), "Exists", "", rnd.choice(["", "PreferNoSchedule", "NoSchedule"]))
                             for _ in range(rnd.randint(1, 2))]
    weight = rnd.choice([0, 3])
    opts = [o for t in tiers for o in t]
    no = next((o for o in opts if o.name == "nodeorder"), None)
    if no is None:
        no = PluginOption.defaults("nodeorder")
        tiers[-1].append(no)
    no.arguments["tainttoleration.weight"] = weight
    if not any(o.name == "predicates" for o in opts) and rnd.random() < 0.7:  # NoSchedule taints reject nodes only here
        tiers[-1].append(PluginOption.defaults("predicates"))
    if "preempt" not in actions:
        actions = actions + ("preempt",)
    if rnd.random() < 0.5:
        conf.update(percentage_nodes_to_find=rnd.choice([34, 50, 67]), min_nodes_to_find=1,
                    last_processed_node_index=rnd.randint(0, 2 * len(tc.Nodes)), enable_predicate_error_cache=False)
    return tc, tiers, actions, conf


def make_guard_case(seed):
    """The pdb and cdp plugins: make_case's clusters (make_topo_case's in a third) widened to 2-30 nodes, running pods with
    labels app / tier or none, 1-4 PDBs with budgets 0-3 over overlapping selectors (some pods in DisruptedPods),
    volcano.sh/cooldown-time on a third of the running pods with PodScheduled times on both sides of the cooldown's end,
    pdb and cdp inserted at random places in the tiers (the last voter of a tier included), feasible-node sampling in half
    the cases. -> (TestCommonStruct, tiers, actions, conf keyword arguments)."""
    from volcano_b200.api import BuildPDB
    rnd = random.Random(seed * 7919 + 29)
    topo = rnd.random() < 0.33
    tc, tiers, actions, conf = make_topo_case(seed) if topo else (*make_case(seed), {})
    for i in range(len(tc.Nodes), rnd.randint(max(2, len(tc.Nodes)), 30)):
        tc.Nodes.append(BuildNode(f"n{i}", BuildResourceList(str(rnd.choice([1, 2, 3, 4])), rnd.choice(["4G", "8G", "16G"]),
                                                               ("pods", str(rnd.choice([3, 6, 20]))))))
    now = 10 ** 18
    running = [p for p in tc.Pods if p.node_name]
    for p in running:
        if rnd.random() < 0.8:
            p.labels = dict(p.labels)
            p.labels["app"] = rnd.choice(["a", "b"])
            if rnd.random() < 0.5:
                p.labels["tier"] = rnd.choice(["x", "y"])
        if rnd.random() < 0.35:
            cool = rnd.choice([60, 600, 3600])
            where = p.labels if (p.labels and rnd.random() < 0.5) else p.annotations
            where["volcano.sh/cooldown-time"] = rnd.choice([f"{cool}s", f"{cool}s", "bogus"])
            p.scheduled_time = now - cool * 10 ** 9 + rnd.choice([-5, 0, 5]) * 10 ** 9
    selectors = [{"app": "a"}, {"app": "b"}, {"tier": "x"}, {"app": "a", "tier": "y"}, {}]
    ns = tc.Pods[0].namespace if tc.Pods else "default"
    pdbs = []
    for i in range(rnd.randint(1, 4)):
        disrupted = [p.name for p in running if rnd.random() < 0.1]
        pdbs.append(BuildPDB(ns, f"pdb{i}", rnd.choice(selectors), rnd.randint(0, 3), disrupted))
    tc.PDBs = pdbs
    for name in ("pdb", "cdp"):
        if rnd.random() < 0.8:
            t = rnd.randrange(len(tiers))
            tiers[t].insert(rnd.randint(0, len(tiers[t])), PluginOption.defaults(name))
    if not any(o.name in ("pdb", "cdp") for t in tiers for o in t):
        tiers[-1].append(PluginOption.defaults("pdb"))
    actions = tuple(a for a in actions if a != "allocate" or rnd.random() < 0.5)
    if not any(a in ("preempt", "reclaim") for a in actions):
        actions = actions + ("preempt",)
    conf["now_ns"] = now
    if rnd.random() < 0.5:
        conf.update(percentage_nodes_to_find=rnd.choice([34, 50, 67]), min_nodes_to_find=1,
                    last_processed_node_index=rnd.randint(0, 2 * len(tc.Nodes)), enable_predicate_error_cache=False)
    return tc, tiers, actions, conf


def make_nta_case(seed):
    """The network-topology-aware plugin: the clusters of make_guard_case (pdb / cdp, the topology-aware reading, sampling),
    make_soft_case (PreferNoSchedule taints) or make_samp_case, widened to at least 4 nodes, under a HyperNode tree of
    1- to 4-node leaves (tier 1; some nodes in no leaf), two tier-2 halves and, often, a tier-3 root; a third of the jobs,
    running or pending, in soft network-topology mode; the plugin in a random tier with random weights, fading 0 / 0.5
    / 0.8, and hypernode binpacking of normal pods on in most cases. -> (TestCommonStruct, tiers, actions, conf)."""
    from volcano_b200.api import BuildHyperNode
    rnd = random.Random(seed * 104651 + 17)
    family = rnd.random()
    if family < 0.4:
        tc, tiers, actions, conf = make_guard_case(seed)
    elif family < 0.7:
        tc, tiers, actions, conf = make_soft_case(seed)
    else:
        tc, tiers, actions, conf = make_samp_case(seed)
    for i in range(len(tc.Nodes), 4):
        tc.Nodes.append(BuildNode(f"n{i}", BuildResourceList(str(rnd.choice([2, 3, 4])), rnd.choice(["4G", "8G", "16G"]),
                                                               ("pods", str(rnd.choice([3, 6, 20]))))))
    names = [n.name for n in tc.Nodes]
    rnd.shuffle(names)
    leaves, i = [], 0
    while i < len(names):
        k = rnd.randint(1, 4)
        if rnd.random() < 0.85:  # the other nodes belong to no leaf: FullScore on tier 1
            leaves.append(BuildHyperNode(f"leaf{len(leaves)}", 1, [(m, "Node") for m in names[i:i + k]]))
        i += k
    hypernodes = list(leaves)
    if len(leaves) >= 2 and rnd.random() < 0.8:
        half = len(leaves) // 2
        hypernodes.append(BuildHyperNode("midA", 2, [(h.name, "HyperNode") for h in leaves[:half]]))
        hypernodes.append(BuildHyperNode("midB", 2, [(h.name, "HyperNode") for h in leaves[half:]]))
        if rnd.random() < 0.6:
            hypernodes.append(BuildHyperNode("root", 3, [("midA", "HyperNode"), ("midB", "HyperNode")]))
    tc.HyperNodes = hypernodes
    for pg in tc.PodGroups:
        if rnd.random() < 0.33:
            pg.network_topology_mode = "soft"
            pg.__post_init__()
    args = {"weight": rnd.choice([1, 10]), "hypernode.binpack.cpu": rnd.choice([1, 5]),
            "hypernode.binpack.memory": rnd.choice([0, 1, 2]),
            "hypernode.binpack.normal-pod.enable": rnd.random() < 0.85,
            "hypernode.binpack.normal-pod.fading": rnd.choice([0, 0.5, 0.8])}
    t = rnd.randrange(len(tiers))
    tiers[t].insert(rnd.randint(0, len(tiers[t])), PluginOption.defaults("network-topology-aware", args))
    if not any(a in ("preempt", "reclaim") for a in actions):
        actions = actions + ("preempt",)
    return tc, tiers, actions, conf


def without_nta(tiers):
    """The tiers without the network-topology-aware plugin."""
    return [[o for o in t if o.name != "network-topology-aware"] for t in tiers if any(o.name != "network-topology-aware" for o in t)]


def _plugins_and_actions(rnd):
    voters = [n for n in ("conformance", "gang", "priority", "drf", "proportion") if rnd.random() < 0.75]
    scorers = [n for n in ("predicates", "nodeorder", "binpack") if rnd.random() < 0.5]
    chosen = voters + scorers
    rnd.shuffle(chosen)
    if not chosen:
        chosen = ["gang"]
    split = rnd.randint(0, len(chosen))
    args = {"binpack": {"binpack.weight": rnd.choice([1, 5]), "binpack.cpu": rnd.choice([1, 3])}}
    tiers = [t for t in ([PluginOption.defaults(n, args.get(n)) for n in chosen[:split]],
                         [PluginOption.defaults(n, args.get(n)) for n in chosen[split:]]) if t]
    actions = tuple(a for a in ("allocate", "preempt", "reclaim") if rnd.random() < 0.7) or ("preempt",)
    if rnd.random() < 0.3:
        actions = ("enqueue",) + actions
    if rnd.random() < 0.2 and "preempt" in actions and "reclaim" in actions:
        actions = tuple(a for a in actions if a not in ("preempt", "reclaim")) + ("reclaim", "preempt")
    return tiers, actions


def compare(res, ref, seed):
    import numpy as np
    for name in ("preempt", "reclaim"):
        a, b = getattr(res, name), getattr(ref, name)
        assert (a is None) == (b is None), (seed, name)
        if a is None:
            continue
        assert np.array_equal(a.visits, b.visits), (seed, name, a.visits, b.visits)
        for f in ("task", "node", "kind", "visit"):
            assert np.array_equal(a.decisions[f], b.decisions[f]), (seed, name, f, a.decisions, b.decisions)
    assert np.array_equal(res.decisions, ref.decisions), seed
    assert np.array_equal(res.visits, ref.visits), seed
    return sum(len(getattr(ref, n).decisions) for n in ("preempt", "reclaim") if getattr(ref, n) is not None)


if __name__ == "__main__":
    import numpy as np
    from oracle.pyoracle import OracleSession
    from volcano_b200 import engine
    from volcano_b200.uthelper import AllocateResult
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
    first, last = int(sys.argv[1]), int(sys.argv[2])
    engine.init(0)
    import conftest  # the oracle engine of the test suite
    oracle = conftest.oracle_engine.__wrapped__() if hasattr(conftest.oracle_engine, "__wrapped__") else None
    ops = evictions = 0
    for seed in range(first, last):
        tc, tiers, actions = make_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = oracle(snap)
        res = engine.gpu_engine(snap)
        ops += compare(res, ref, seed)
    print(f"seeds [{first},{last}): {ops} evict/pipeline operations identical")
