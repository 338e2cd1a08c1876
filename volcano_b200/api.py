"""Host-side mirror of the reference's cluster objects and unit-test builders.

The reference's action tests are written against literal v1.Pod / v1.Node / PodGroup /
Queue objects built with util.BuildNode/BuildPod/BuildPodGroup/BuildQueue
(pkg/scheduler/util/test_utils.go:43-97,336-351,466-479) and api.BuildResourceList
(pkg/scheduler/api/test_utils.go:102-118).  The same shapes and names are kept here so
that parity tests read like the reference's own tests; `snapshot.encode_cluster` turns
them into the structure-of-arrays the C ABI takes (what the cgo shim does in Go).
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Sequence, Dict, List, Optional, Tuple

# ---------------------------------------------------------------------------------------
# resource.Quantity (k8s.io/apimachinery/pkg/api/resource): only Value()/MilliValue()
# ---------------------------------------------------------------------------------------
_BIN = {"Ki": 2**10, "Mi": 2**20, "Gi": 2**30, "Ti": 2**40, "Pi": 2**50, "Ei": 2**60}
_DEC = {"n": (1, 10**9), "u": (1, 10**6), "m": (1, 1000), "": (1, 1), "k": (10**3, 1), "M": (10**6, 1),
        "G": (10**9, 1), "T": (10**12, 1), "P": (10**15, 1), "E": (10**18, 1)}
_QRE = re.compile(r"^([+-]?[0-9]*\.?[0-9]*)([eE][+-]?[0-9]+|[a-zA-Z]*)$")


def parse_quantity(s) -> Tuple[int, int]:
    """-> (numerator, denominator) of the exact value."""
    if isinstance(s, (int, float)):
        s = repr(s) if isinstance(s, float) else str(s)
    m = _QRE.match(str(s).strip())
    if not m or m.group(1) in ("", "+", "-", "."):
        raise ValueError(f"bad quantity {s!r}")
    num_s, suf = m.group(1), m.group(2)
    if "." in num_s:
        ip, fp = num_s.split(".")
        num = int((ip or "0") + fp) if ip not in ("-", "+") else int(ip + "0" + fp)
        den = 10 ** len(fp)
    else:
        num, den = int(num_s), 1
    if suf in _BIN:
        num *= _BIN[suf]
    elif suf in _DEC:
        a, b = _DEC[suf]
        num *= a
        den *= b
    elif suf[:1] in ("e", "E"):
        e = int(suf[1:])
        if e >= 0:
            num *= 10**e
        else:
            den *= 10 ** (-e)
    else:
        raise ValueError(f"bad quantity suffix {s!r}")
    return num, den


def _ceil_div(a: int, b: int) -> int:
    return -((-a) // b)


def quantity_value(s) -> int:  # Quantity.Value(): rounds up
    n, d = parse_quantity(s)
    return _ceil_div(n, d)


def quantity_milli(s) -> int:  # Quantity.MilliValue(): rounds up
    n, d = parse_quantity(s)
    return _ceil_div(n * 1000, d)


ResourceList = Dict[str, str]


def BuildResourceList(cpu: str, memory: str, *scalars: Tuple[str, str]) -> ResourceList:
    """api.BuildResourceList (pkg/scheduler/api/test_utils.go:102-118)."""
    rl = {"cpu": cpu, "memory": memory}
    for name, value in scalars:
        rl[name] = value
    return rl


def BuildResourceListWithGPU(cpu: str, memory: str, gpu: str, *scalars: Tuple[str, str]) -> ResourceList:
    rl = BuildResourceList(cpu, memory, *scalars)
    rl["nvidia.com/gpu"] = gpu
    return rl


# ---------------------------------------------------------------------------------------
# v1.Node / v1.Pod / PodGroup / Queue (just the fields the allocate path reads)
# ---------------------------------------------------------------------------------------
@dataclass
class Taint:
    key: str
    value: str = ""
    effect: str = "NoSchedule"  # NoSchedule | PreferNoSchedule | NoExecute


@dataclass
class Toleration:
    key: str = ""
    operator: str = "Equal"  # Equal | Exists
    value: str = ""
    effect: str = ""  # "" matches every effect

    def tolerates(self, t: Taint) -> bool:
        # v1.Toleration.ToleratesTaint (k8s.io/api/core/v1/toleration.go)
        if self.effect and self.effect != t.effect:
            return False
        if self.key and self.key != t.key:
            return False
        if self.operator == "Exists":
            return True
        return self.value == t.value


@dataclass
class NodeSelectorRequirement:
    key: str
    operator: str  # In | NotIn | Exists | DoesNotExist | Gt | Lt
    values: Tuple[str, ...] = ()

    def matches(self, labels: Dict[str, str]) -> bool:
        has = self.key in labels
        v = labels.get(self.key)
        op = self.operator
        if op == "In":
            return has and v in self.values
        if op == "NotIn":
            return not (has and v in self.values)
        if op == "Exists":
            return has
        if op == "DoesNotExist":
            return not has
        if op in ("Gt", "Lt"):
            if not has:
                return False
            try:
                lv, rv = int(v), int(self.values[0])
            except (ValueError, IndexError):
                return False
            return lv > rv if op == "Gt" else lv < rv
        raise ValueError(op)

    def ident(self):
        return (self.key, self.operator, tuple(self.values))


PREEMPTABLE_KEY = "volcano.sh/preemptable"
REVOCABLE_ZONE = "volcano.sh/revocable-zone"  # v1beta1.RevocableZone


@dataclass
class Node:
    name: str
    allocatable: ResourceList
    labels: Dict[str, str] = field(default_factory=dict)
    taints: List[Taint] = field(default_factory=list)
    unschedulable: bool = False
    annotations: Dict[str, str] = field(default_factory=dict)
    revocable_zone: str = ""  # label volcano.sh/revocable-zone

    def __post_init__(self):
        if not self.revocable_zone:  # setRevocableZone, api/node_info.go:252-265
            self.revocable_zone = self.labels.get(REVOCABLE_ZONE, "")


@dataclass
class Pod:
    namespace: str
    name: str
    node_name: str
    phase: str  # Pending | Running | Succeeded | Failed | Unknown
    requests: ResourceList
    group_name: str
    labels: Dict[str, str] = field(default_factory=dict)
    node_selector: Dict[str, str] = field(default_factory=dict)
    annotations: Dict[str, str] = field(default_factory=dict)
    tolerations: List[Toleration] = field(default_factory=list)
    # required nodeAffinity: OR over terms, AND inside a term
    affinity_required: List[List[NodeSelectorRequirement]] = field(default_factory=list)
    # preferred nodeAffinity: (weight, AND-list)
    affinity_preferred: List[Tuple[int, List[NodeSelectorRequirement]]] = field(default_factory=list)
    priority: Optional[int] = None
    creation_ts: int = 0
    deleting: bool = False
    uid: str = ""
    preemptable: bool = False
    revocable_zone: str = ""  # annotation volcano.sh/revocable-zone
    preemption_policy: str = ""    # pod.Spec.PreemptionPolicy ("Never": the pod never preempts / reclaims)
    priority_class_name: str = ""  # pod.Spec.PriorityClassName (conformance: system-*-critical pods are never evicted)
    nominated_node_name: str = ""  # pod.Status.NominatedNodeName (left by a preemption of an earlier cycle, allocate.go:624-634)
    start_time: Optional[int] = None  # pod.Status.StartTime in ns since the epoch (None: not started)
    scheduled_time: Optional[int] = None  # LastTransitionTime of the first PodScheduled=True condition, ns (None: none)

    def __post_init__(self):
        if not self.uid:
            self.uid = f"{self.namespace}-{self.name}"  # util/test_utils.go:74
        if not self.revocable_zone:  # GetPodRevocableZone, api/pod_info.go:153-165
            if REVOCABLE_ZONE in self.annotations:  # only the wildcard zone is honoured
                self.revocable_zone = "*" if self.annotations[REVOCABLE_ZONE] == "*" else ""
            elif self.annotations.get("volcano.sh/preemptable", "").lower() in ("1", "t", "true"):
                self.revocable_zone = "*"

    @property
    def key(self) -> str:
        return f"{self.namespace}/{self.name}"


@dataclass
class PodGroup:
    name: str
    namespace: str
    queue: str
    min_member: int
    min_task_member: Optional[Dict[str, int]] = None
    phase: str = "Inqueue"  # Pending | Inqueue | Running | ...
    priority: int = 0  # resolved PriorityClass value (cache/cache.go:1526-1532)
    creation_ts: int = 0
    preemptable: bool = False
    unsupported: bool = False  # hard network topology / subGroupPolicy
    network_topology_mode: str = ""  # "" | "soft" | "hard" (Spec.NetworkTopology.Mode)
    allocated_hypernode: str = ""    # volcano.sh/job-allocated-hypernode: AllocatedHyperNode carried into the session

    def __post_init__(self):
        if self.network_topology_mode == "hard":
            self.unsupported = True


@dataclass
class Queue:
    name: str
    weight: int = 1
    capability: Optional[ResourceList] = None
    guarantee: Optional[ResourceList] = None
    priority: int = 0
    state: str = "Open"
    creation_ts: int = 0
    reclaimable: bool = True  # Queue.Spec.Reclaimable (nil = true, api/queue_info.go:80-95)
    hierarchy: str = ""  # volcano.sh/hierarchy annotation (QueueInfo.Hierarchy, api/queue_info.go:60)
    weights: str = ""    # volcano.sh/hierarchy-weights annotation (QueueInfo.Weights, api/queue_info.go:61)


@dataclass
class HyperNode:
    """topology.volcano.sh HyperNode (api.BuildHyperNode, api/test_utils.go): members are (name, type) with
    type "Node" or "HyperNode"; only the exact-match selector is modelled."""
    name: str
    tier: int
    members: List[Tuple[str, str]] = field(default_factory=list)


def BuildHyperNode(name: str, tier: int, members: Sequence[Tuple[str, str]]) -> HyperNode:
    return HyperNode(name=name, tier=tier, members=[(m[0], m[1]) for m in members])


@dataclass
class PodDisruptionBudget:
    """policy/v1 PodDisruptionBudget as the pdb plugin reads it (plugins/pdb/pdb.go:65-126): the selector's matchLabels
    (None or empty: a nil or empty selector, which matches nothing), Status.DisruptionsAllowed and the names in
    Status.DisruptedPods."""
    namespace: str
    name: str
    match_labels: Optional[Dict[str, str]] = None
    disruptions_allowed: int = 0
    disrupted_pods: List[str] = field(default_factory=list)

    def counts(self, pod: "Pod") -> bool:
        """Whether this PDB takes one from its budget when the plugin walks `pod` (a pod with labels)."""
        return (self.namespace == pod.namespace and bool(self.match_labels)
                and all(pod.labels.get(k) == v for k, v in self.match_labels.items())
                and pod.name not in self.disrupted_pods)


def BuildPDB(namespace: str, name: str, match_labels: Optional[Dict[str, str]], disruptions_allowed: int,
             disrupted_pods: Sequence[str] = ()) -> PodDisruptionBudget:
    return PodDisruptionBudget(namespace, name, dict(match_labels) if match_labels is not None else None,
                               disruptions_allowed, list(disrupted_pods))


COOLDOWN_TIME_KEY = "volcano.sh/cooldown-time"  # v1beta1.CooldownTime

_DURATION_UNITS = {"ns": 1, "us": 1000, "\u00b5s": 1000, "\u03bcs": 1000, "ms": 10 ** 6, "s": 10 ** 9, "m": 60 * 10 ** 9,
                   "h": 3600 * 10 ** 9}
_DURATION_RE = re.compile(r"([0-9]*(?:\.[0-9]*)?)([a-z\u00b5\u03bc]+)")


def go_parse_duration(text: str) -> Optional[int]:
    """time.ParseDuration in ns, None where it returns an error."""
    s = text
    neg = False
    if s[:1] in ("-", "+"):
        neg, s = s[0] == "-", s[1:]
    if s == "0":
        return 0
    if not s:
        return None
    total, pos = 0, 0
    while pos < len(s):
        m = _DURATION_RE.match(s, pos)
        if not m or m.group(1) in ("", ".") or m.group(2) not in _DURATION_UNITS:
            return None
        whole, _, frac = m.group(1).partition(".")
        unit = _DURATION_UNITS[m.group(2)]
        v = int(whole or "0") * unit
        if frac:
            scale = 1
            f = 0
            for ch in frac:  # the fraction is truncated to whole nanoseconds, as Go's leadingFraction + float scaling
                if scale >= 10 ** 18:
                    break
                f = f * 10 + int(ch)
                scale *= 10
            v += int(f * (unit / scale))
        total += v
        if total > 2 ** 63 - 1 + (1 if neg else 0):
            return None
        pos = m.end()
    return -total if neg else total


def pod_cooldown_until(pod: "Pod") -> Optional[int]:
    """cdp's protection end (plugins/cdp/cdp.go:56-96): the cooldown from the label, else the annotation (an unparsable
    label disables it); only a Running pod with a PodScheduled=True condition is protected; None: never protected."""
    v = pod.labels.get(COOLDOWN_TIME_KEY, pod.annotations.get(COOLDOWN_TIME_KEY))
    if v is None:
        return None
    d = go_parse_duration(v)
    if d is None or pod.phase != "Running" or pod.scheduled_time is None:
        return None
    return pod.scheduled_time + d


TASK_SPEC_KEY = "volcano.sh/task-spec"  # batch.TaskSpecKey
TASK_PRIORITY_ANNOTATION = "volcano.sh/task-priority"


def BuildNode(name: str, alloc: ResourceList, labels: Optional[Dict[str, str]] = None) -> Node:
    return Node(name=name, allocatable=dict(alloc), labels=dict(labels or {}))


def BuildPod(namespace, name, node_name, phase, req, group_name, labels=None, selector=None) -> Pod:
    return Pod(namespace=namespace, name=name, node_name=node_name, phase=phase, requests=dict(req or {}),
               group_name=group_name, labels=dict(labels or {}), node_selector=dict(selector or {}))


def pod_preemptable(pod: "Pod") -> bool:
    """GetPodPreemptable, api/pod_info.go:125-151: annotation, then label volcano.sh/preemptable (strconv.ParseBool);
    absent = true."""
    for src in (pod.annotations, pod.labels):
        if PREEMPTABLE_KEY in src:
            v = str(src[PREEMPTABLE_KEY])
            if v in ("1", "t", "T", "TRUE", "true", "True"):
                return True
            return False  # "0", "f", ... and unparsable values
    return True


def pod_critical(pod: "Pod") -> bool:
    """conformance evictableFn, plugins/conformance/conformance.go:50-56."""
    return pod.priority_class_name in ("system-cluster-critical", "system-node-critical") or pod.namespace == "kube-system"


def BuildPodWithPreemptionPolicy(namespace, name, node_name, phase, req, group_name, labels=None, selector=None,
                                 preemption_policy: str = "") -> Pod:
    """util/test_utils.go:328-333."""
    p = BuildPod(namespace, name, node_name, phase, req, group_name, labels, selector)
    p.preemption_policy = preemption_policy
    return p


def BuildPodWithPriority(namespace, name, node_name, phase, req, group_name, labels=None, selector=None,
                         priority: Optional[int] = None) -> Pod:
    """util/test_utils.go:128-158."""
    p = BuildPod(namespace, name, node_name, phase, req, group_name, labels, selector)
    p.priority = priority
    return p


def BuildPodGroupWithPrio(name, ns, queue, min_member, task_min_member, phase, priority: int) -> "PodGroup":
    """util/test_utils.go:368-382; `priority` is the resolved PriorityClass value (cache/cache.go:1526-1532)."""
    pg = BuildPodGroup(name, ns, queue, min_member, task_min_member, phase)
    pg.priority = priority
    return pg


def BuildPodGroup(name, ns, queue, min_member, task_min_member=None, phase="Inqueue") -> PodGroup:
    return PodGroup(name=name, namespace=ns, queue=queue, min_member=min_member,
                    min_task_member=dict(task_min_member) if task_min_member else None, phase=phase)


def BuildPodGroupWithNetWorkTopologies(name, ns, hypernode_name, queue, min_member, task_min_member, phase, mode,
                                       highest_tier_allowed) -> PodGroup:
    """util/test_utils.go:393-402."""
    pg = BuildPodGroup(name, ns, queue, min_member, task_min_member, phase)
    pg.network_topology_mode = mode
    pg.allocated_hypernode = hypernode_name
    pg.__post_init__()
    return pg


def BuildQueue(name, weight, cap=None) -> Queue:
    return Queue(name=name, weight=weight, capability=dict(cap) if cap else None)


KUBE_HIERARCHY_ANNOTATION_KEY = "volcano.sh/hierarchy"
KUBE_HIERARCHY_WEIGHT_ANNOTATION_KEY = "volcano.sh/hierarchy-weights"


def BuildQueueWithAnnos(name, weight, cap=None, annos=None) -> Queue:
    """util.BuildQueueWithAnnos: a queue whose annotations carry the hdrf hierarchy and its weights."""
    annos = annos or {}
    return Queue(name=name, weight=weight, capability=dict(cap) if cap else None,
                 hierarchy=annos.get(KUBE_HIERARCHY_ANNOTATION_KEY, ""),
                 weights=annos.get(KUBE_HIERARCHY_WEIGHT_ANNOTATION_KEY, ""))


def get_task_role(pod: Pod) -> str:
    """getTaskRole, api/job_info.go:166-179."""
    ts = pod.annotations.get(TASK_SPEC_KEY, "")
    if ts:
        return ts
    return pod.labels.get(TASK_SPEC_KEY, "") or ""


def get_task_status(pod: Pod) -> str:
    """getTaskStatus, api/helpers.go:41-67."""
    if pod.phase == "Running":
        return "Releasing" if pod.deleting else "Running"
    if pod.phase == "Pending":
        if pod.deleting:
            return "Releasing"
        return "Pending" if not pod.node_name else "Bound"
    if pod.phase == "Succeeded":
        return "Succeeded"
    if pod.phase == "Failed":
        return "Failed"
    return "Unknown"


def allocated_status(st: str) -> bool:  # api/helpers.go:80-87
    return st in ("Bound", "Binding", "Running", "Allocated")


def pod_index_under_task(name: str) -> int:
    """GetPodIndexUnderTask + strconv.Atoi (pkg/controllers/job/helpers/helpers.go:44-57); -1 = not numeric."""
    parts = name.split("-")
    if len(parts) >= 3:
        s = parts[-1]
        if re.fullmatch(r"[+-]?[0-9]+", s):
            v = int(s)
            return v if v >= 0 else -1  # negative indices never occur; keep -1 as the error marker
    return -1
