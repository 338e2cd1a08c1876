"""API-level differential fuzzing: random small clusters built from the host mirror of the reference's objects
(labels, selectors, required / preferred node affinity, taints of all effects, tolerations, tdm revocable zones,
running pods, releasing resources via deleting pods, task roles + TaskMinAvailable, queue weights / capabilities /
priorities, HyperNode trees with soft-mode topology jobs, random plugin sets and arguments) — CUDA path vs CPU oracle.
Test infrastructure (imports the oracle).  Usage: python tools/fuzz_api.py [n_cases] [first_seed]"""
import os
import random
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.pyoracle import OracleSession  # noqa: E402
from volcano_b200 import engine  # noqa: E402
from volcano_b200.api import (BuildHyperNode, BuildNode, BuildPod, BuildPodGroup, BuildPodGroupWithNetWorkTopologies,  # noqa: E402
                              BuildQueue, BuildResourceList, NodeSelectorRequirement, Taint, Toleration)
from volcano_b200.snapshot import PluginOption  # noqa: E402
from volcano_b200.uthelper import TestCommonStruct  # noqa: E402

ZONES = ["za", "zb", "zc"]
POOLS = ["p0", "p1"]


def make_case(seed, big=False):
    rnd = random.Random(seed)
    rnd2 = random.Random(seed * 7919 + 13)  # later additions draw from their own stream: earlier seeds keep their clusters
    mix_names = rnd2.random() < 0.3  # jobs mixing pods with and without a numeric name index (CompareTask is intransitive there)
    rnd3 = random.Random(seed * 104729 + 7)  # a third stream: nominated nodes (one case in eight)
    nominate = rnd3.random() < 0.125
    be_p = rnd.choice([0.05, 0.05, 0.3])  # share of BestEffort pods (the backfill action's tasks)
    n_nodes = rnd.randint(3, 40) if not big else rnd.randint(40, 400)
    nodes = []
    leaves = rnd.randint(2, 5) if not big else rnd.randint(3, 12)
    for i in range(n_nodes):
        cpu = rnd.choice(["4", "8", "16", "32"])
        mem = rnd.choice(["8Gi", "16Gi", "64Gi"])
        extra = [("pods", str(rnd.choice([3, 5, 10, 110])))]
        if rnd.random() < 0.4:
            extra.append(("nvidia.com/gpu", str(rnd.choice([2, 4, 8]))))
        if rnd.random() < 0.3:
            extra.append(("example.com/foo", str(rnd.choice([4, 16]))))
        labels = {"zone": rnd.choice(ZONES), "pool": rnd.choice(POOLS)}
        if rnd.random() < 0.3:
            labels["tier"] = str(rnd.randint(1, 9))
        if rnd.random() < 0.2:
            labels["volcano.sh/revocable-zone"] = rnd.choice(["rz1", "rz2"])
        n = BuildNode(f"n{i:02d}", BuildResourceList(cpu, mem, *extra), labels)
        for _ in range(rnd.choice([0, 0, 0, 1, 2])):
            n.taints.append(Taint(rnd.choice(["dedicated", "gpu", "spot"]), rnd.choice(["a", "b"]),
                                  rnd.choice(["NoSchedule", "PreferNoSchedule", "NoExecute"])))
        if rnd.random() < 0.05:
            n.unschedulable = True
        nodes.append(n)
    n_queues = rnd.randint(1, 4)
    queues = []
    for q in range(n_queues):
        cap = BuildResourceList(str(rnd.choice([8, 16, 64])), rnd.choice(["16Gi", "64Gi", "256Gi"])) if rnd.random() < 0.3 else None
        qu = BuildQueue(f"q{q}", rnd.randint(1, 4), cap)
        qu.priority = rnd.choice([0, 0, 1, 5])
        if rnd.random() < 0.08:
            qu.state = "Closed"
        if rnd.random() < 0.15:
            qu.guarantee = BuildResourceList(str(rnd.choice([1, 4])), rnd.choice(["2Gi", "8Gi"]))
        queues.append(qu)
    use_topo = rnd.random() < 0.5
    hypernodes = None
    if use_topo:
        hypernodes = []
        per = max(1, n_nodes // leaves)
        for l in range(leaves):
            members = [(f"n{i:02d}", "Node") for i in range(l * per, min(n_nodes, (l + 1) * per))]
            if members:
                hypernodes.append(BuildHyperNode(f"leaf{l}", 1, members))
        if len(hypernodes) >= 2 and rnd.random() < 0.8:
            half = len(hypernodes) // 2
            hypernodes.append(BuildHyperNode("midA", 2, [(h.name, "HyperNode") for h in hypernodes[:half]]))
            hypernodes.append(BuildHyperNode("midB", 2, [(h.name, "HyperNode") for h in hypernodes[half:-1] if h.tier == 1]))
            if rnd.random() < 0.6:
                hypernodes.append(BuildHyperNode("root", 3, [("midA", "HyperNode"), ("midB", "HyperNode")]))
    pods, pgs = [], []
    n_jobs = rnd.randint(1, 8) if not big else rnd.randint(5, 40)
    for j in range(n_jobs):
        size = rnd.choice([1, 1, 2, 3, 4, 6, 8]) if not big else rnd.choice([1, 2, 4, 8, 16, 32])
        min_member = rnd.choice([1, size, max(1, size // 2), size + (1 if rnd.random() < 0.1 else 0)])
        roles = rnd.random() < 0.3 and size >= 2
        tmm = {"master": 1, "worker": max(0, min_member - 1)} if roles and rnd.random() < 0.7 else None
        qname = f"q{rnd.randrange(n_queues)}"
        phase = rnd.choice(["Inqueue", "Inqueue", "Running", "Pending"])
        if use_topo and rnd.random() < 0.4:
            pg = BuildPodGroupWithNetWorkTopologies(f"pg{j}", "ns", "", qname, min_member, tmm, phase, "soft", 0)
        else:
            pg = BuildPodGroup(f"pg{j}", "ns", qname, min_member, tmm, phase)
        pg.priority = rnd.choice([0, 0, 1, 2])
        pg.preemptable = rnd.random() < 0.2
        pg.creation_ts = rnd.randint(0, 5)
        pgs.append(pg)
        req = BuildResourceList(rnd.choice(["500m", "1", "2", "4"]), rnd.choice(["1Gi", "2Gi", "8Gi"]),
                                *([("nvidia.com/gpu", str(rnd.choice([1, 2])))] if rnd.random() < 0.25 else []),
                                *([("example.com/foo", "1")] if rnd.random() < 0.15 else []))
        sel = {"zone": rnd.choice(ZONES)} if rnd.random() < 0.25 else {}
        for k in range(size):
            role = ("master" if k == 0 else "worker") if roles else "worker"
            running = rnd.random() < 0.2
            node_name = rnd.choice(nodes).name if running else ""
            p = BuildPod("ns", f"j{j}-{role}-{k}", node_name, "Running" if running else "Pending",
                         req if role == "worker" or rnd.random() < 0.5 else BuildResourceList("1", "1Gi"),
                         f"pg{j}", {"volcano.sh/task-spec": role}, sel)
            if mix_names and rnd2.random() < 0.4:
                p.name = f"j{j}-{role}-x{k}"  # no numeric suffix: ordered by creation time, then UID
                p.uid = f"ns-{p.name}"
                p.creation_ts = rnd2.randint(0, 3)
            elif mix_names:
                p.creation_ts = rnd2.randint(0, 3)
            if rnd.random() < 0.3:
                p.tolerations.append(Toleration(rnd.choice(["dedicated", "gpu", "spot", ""]), rnd.choice(["Equal", "Exists"]),
                                                rnd.choice(["a", "b"]), rnd.choice(["", "NoSchedule", "PreferNoSchedule"])))
            if rnd.random() < 0.15:
                p.affinity_required.append([NodeSelectorRequirement("pool", rnd.choice(["In", "NotIn"]), (rnd.choice(POOLS),))])
                if rnd.random() < 0.5:
                    p.affinity_required.append([NodeSelectorRequirement("tier", rnd.choice(["Gt", "Lt", "Exists", "DoesNotExist"]), ("5",))])
            if rnd.random() < 0.2:
                p.affinity_preferred.append((rnd.randint(1, 100), [NodeSelectorRequirement("zone", "In", (rnd.choice(ZONES),))]))
            if rnd.random() < 0.15:
                p.annotations["volcano.sh/revocable-zone"] = "*"
                p.__post_init__()
            if running and rnd.random() < 0.3:
                p.deleting = True  # Releasing on its node
            if rnd.random() < 0.2:
                p.priority = rnd.randint(0, 3)
            if rnd.random() < be_p:
                p.requests = {}  # BestEffort: stays out of the allocate action, counts as pending best-effort
            if nominate and not running and rnd3.random() < 0.3:  # Status.NominatedNodeName, allocate.go:624-634
                p.nominated_node_name = rnd3.choice(nodes).name if rnd3.random() < 0.9 else "no-such-node"
            pods.append(p)
    # plugin set
    names = ["priority", "gang", "drf", "predicates", "proportion", "nodeorder", "binpack", "tdm", "network-topology-aware"]
    chosen = [n for n in names if rnd.random() < 0.75]
    want_backfill = rnd.random() < 0.7
    if "gang" not in chosen and rnd.random() < 0.7:
        chosen.append("gang")
    args = {
        "binpack": {"binpack.weight": rnd.choice([1, 5, 10]), "binpack.cpu": rnd.choice([1, 5]), "binpack.memory": rnd.choice([1, 2]),
                    "binpack.resources": "nvidia.com/gpu, example.com/foo", "binpack.resources.nvidia.com/gpu": rnd.choice([0, 2, 7])},
        "nodeorder": {"leastrequested.weight": rnd.choice([0, 1, 2, -1]), "mostrequested.weight": rnd.choice([0, 0, 1, -2]),
                      "balancedresource.weight": rnd.choice([0, 1]), "nodeaffinity.weight": rnd.choice([0, 2]),
                      "tainttoleration.weight": rnd.choice([0, 3])},
        "network-topology-aware": {"weight": rnd.choice([1, 10]), "hypernode.binpack.cpu": rnd.choice([1, 5]),
                                   "hypernode.binpack.resources": "nvidia.com/gpu",
                                   "hypernode.binpack.normal-pod.enable": rnd.random() < 0.8,
                                   "hypernode.binpack.normal-pod.fading": rnd.choice([0, 0.5, 0.8])},
        "tdm": {"tdm.revocable-zone.rz1": "0:00-0:00", "tdm.revocable-zone.rz2": "0:00-0:01"},
    }
    split = rnd.randint(0, len(chosen))
    tiers = [t for t in ([PluginOption.defaults(n, args.get(n)) for n in chosen[:split]],
                         [PluginOption.defaults(n, args.get(n)) for n in chosen[split:]]) if t]
    tc = TestCommonStruct(Name=f"fuzz{seed}", Nodes=nodes, Pods=pods, PodGroups=pgs, Queues=queues, HyperNodes=hypernodes,
                          TdmZoneActive={"rz1": rnd.random() < 0.7, "rz2": rnd.random() < 0.3})
    actions = ("enqueue", "allocate") if rnd.random() < 0.5 else ("allocate",)
    if want_backfill:
        actions += ("backfill",)
    tc.conf_kw = {}
    if rnd.random() < 0.3:  # feasible-node sampling with a rotating start index
        tc.conf_kw = dict(percentage_nodes_to_find=rnd.choice([0, 10, 30, 60]), min_nodes_to_find=rnd.choice([1, 3, 10, 50]),
                          min_percentage_nodes_to_find=rnd.choice([5, 20]), last_processed_node_index=rnd.randint(0, 500))
    return tc, tiers, actions


def make_hdrf_case(seed):
    """The hdrf family: a make_case cluster with drf's enableHierarchy on and random volcano.sh/hierarchy annotations —
    trees up to 4 levels below the root, nodes shared by several queues, root-level queues, weights that clamp to 1
    ("0.5", "abc", "0") — and drf before or after proportion. Returns (case, tiers, actions, hierarchy, weights)."""
    tc, tiers, actions = make_case(seed)
    rnd = random.Random(seed * 15485863 + 3)
    opts = [po for t in tiers for po in t]
    if not any(po.name == "drf" for po in opts):
        (tiers[-1] if tiers else tiers.append([]) or tiers[-1]).append(PluginOption.defaults("drf"))
    for t in tiers:
        for po in t:
            if po.name == "drf":
                po.hierarchy = True
        names = [po.name for po in t]
        if "drf" in names and "proportion" in names and rnd.random() < 0.5:  # the other tier order of the chain
            i, k = names.index("drf"), names.index("proportion")
            t[i], t[k] = t[k], t[i]
    segs = ["d0", "d1", "t0", "t1", "t2"]
    for q in tc.Queues:
        depth = rnd.choice([0, 1, 1, 2, 2, 3, 4])
        if depth == 0:
            q.hierarchy, q.weights = rnd.choice([("", ""), ("root", "1")])
            continue
        q.hierarchy = "/".join(["root"] + [rnd.choice(segs) for _ in range(depth)])
        q.weights = "/".join([str(rnd.choice([1, 100]))] + [rnd.choice(["1", "2", "5", "0.5", "abc", "0", "1.5", "0x2p0"])
                                                              for _ in range(depth)])
    return tc, tiers, actions, [q.hierarchy for q in tc.Queues], [q.weights for q in tc.Queues]


def backfill_supported(tiers, conf_kw):
    """vc_backfill_run's documented limit: "pods" must not be a weighted hypernode-binpacking resource."""
    return not any(po.name == "network-topology-aware" and "pods" in str(po.arguments.get("hypernode.binpack.resources", ""))
                   for t in tiers for po in t)


def main():
    n_cases = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    first = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    big = len(sys.argv) > 3 and sys.argv[3] == "big"
    engine.init(0)
    bad = unsupported = dense_bad = bf_bad = bf_runs = bf_placed = 0
    for seed in range(first, first + n_cases):
        tc, tiers, actions = make_case(seed, big)
        if not tiers:
            continue
        snap = tc.RegisterSession(tiers, actions=actions, **tc.conf_kw)
        if snap.T == 0 or snap.N == 0:
            continue
        o = OracleSession(snap, threads=1)
        dec, vis, fe = o.allocate()
        eng = engine.Engine(snap)
        try:
            eng.upload()
            r = eng.allocate()
        except engine.VcError as e:
            unsupported += 1
            o.close()
            eng.close()
            print(f"seed {seed}: {e}")
            continue
        ok = (np.array_equal(dec, r.decisions) and np.array_equal(vis, r.visits) and np.array_equal(fe, r.fit_errors))
        from oracle import pyoracle as _po
        ok = ok and r.stats["last_processed_node_index"] == _po.lib().vco_last_processed_node_index(o.h)
        if snap.hn_job_soft is not None and snap.hn_job_soft.any():
            from oracle import pyoracle
            ja = np.array([pyoracle.lib().vco_job_allocated_hypernode(o.h, j) for j in range(snap.J)], np.int32)
            ok = ok and r.job_allocated_hypernodes is not None and np.array_equal(ja, r.job_allocated_hypernodes)
        if not ok:
            bad += 1
            k = next((i for i in range(min(len(dec), len(r.decisions))) if dec[i] != r.decisions[i]), -1)
            print(f"MISMATCH seed={seed}: oracle {len(dec)} dec / {len(vis)} visits, gpu {len(r.decisions)} / {len(r.visits)}; first diff {k}"
                  + (f" oracle={dec[k]} gpu={r.decisions[k]}" if k >= 0 else ""))
        # the backfill action on the state allocate left
        if "backfill" in actions and snap.B > 0:
            try:
                rb = eng.backfill()
            except engine.VcError as e:
                rb = None
                if e.code != -4:
                    raise
            if rb is not None:
                bdec, bvis, bfe = o.backfill()
                bf_runs += 1
                bf_placed += len(bdec)
                same_idx = rb.stats["last_processed_node_index"] == _po.lib().vco_last_processed_node_index(o.h)
                if not (same_idx and np.array_equal(bdec, rb.decisions) and np.array_equal(bvis, rb.visits) and np.array_equal(bfe, rb.fit_errors)):
                    bf_bad += 1
                    print(f"BACKFILL MISMATCH seed={seed}: oracle {len(bdec)} dec / {len(bvis)} visits / {len(bfe)} fit errors, "
                          f"gpu {len(rb.decisions)} / {len(rb.visits)} / {len(rb.fit_errors)}")
        eng.close()
        # dense pass on the opening snapshot
        o2 = OracleSession(snap)
        om, osc, obs, obn = o2.score_matrix()
        o2.close()
        o.close()
        try:
            e = engine.Engine(snap)
            e.upload()
            m, sc, bs, bn = e.score_matrix()
            e.close()
            if not (np.array_equal(m, om) and np.array_equal(sc, osc) and np.array_equal(bn, obn) and np.array_equal(bs, obs)):
                dense_bad += 1
                print(f"DENSE MISMATCH seed={seed}")
        except engine.VcError:
            pass
    print(f"{n_cases} cases: {bad} allocate mismatches, {dense_bad} dense mismatches, {unsupported} unsupported; "
          f"backfill: {bf_runs} runs, {bf_placed} placements, {bf_bad} mismatches")


if __name__ == "__main__":
    main()
