"""Mirror of the reference's action-test harness, pkg/scheduler/uthelper/helper.go:60-296.

`TestCommonStruct` keeps the reference's field names (Name, Plugins, Pods, Nodes, PodGroups,
Queues, ExpectBindMap, ExpectBindsNum, ExpectPipeLined) so a reference test case can be
transcribed literally.  RegisterSession(tiers) ~ framework.OpenSession with explicit tiers
(helper.go:127-132); Run(engine) ~ action.Execute(ssn) where `engine` is any callable
Snapshot -> AllocateResult (the CUDA engine in volcano_b200.engine, or the CPU oracle in
tests); CheckAll ~ helper.go:239-296 with the FakeBinder (util/test_utils.go:544-588)
replaced by replaying the returned Statement operations.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

from . import abi
from .api import BuildQueueWithAnnos, HyperNode, Node, Pod, PodDisruptionBudget, PodGroup, Queue  # noqa: F401  (util.BuildQueueWithAnnos)
from .snapshot import PluginOption, SchedulerConf, Snapshot, encode_cluster


@dataclass
class AllocateResult:
    decisions: np.ndarray   # structured: task,node,kind,visit,score
    visits: np.ndarray      # structured: job,outcome,first_op,n_ops
    fit_errors: np.ndarray  # int32 task indices
    stats: Optional[dict] = None
    job_allocated_hypernodes: Optional[np.ndarray] = None  # subJob.AllocatedHyperNode after the run (topology sessions)
    backfill: Optional["AllocateResult"] = None  # the backfill action's result (task = index into backfill_task_keys)
    preempt: Optional["AllocateResult"] = None   # the preempt action's result (VC_OP_EVICT: task = index into running_task_keys)
    reclaim: Optional["AllocateResult"] = None   # the reclaim action's result


@dataclass
class TestCommonStruct:
    __test__ = False  # not a pytest class
    Name: str = ""
    Plugins: Optional[dict] = None  # reference: name -> PluginBuilder; informational here
    Pods: List[Pod] = field(default_factory=list)
    Nodes: List[Node] = field(default_factory=list)
    PodGroups: List[PodGroup] = field(default_factory=list)
    Queues: List[Queue] = field(default_factory=list)
    ExpectBindMap: Dict[str, str] = field(default_factory=dict)
    ExpectBindsNum: Optional[int] = None
    ExpectPipeLined: Optional[Dict[str, List[str]]] = None  # job -> node names
    ExpectEvicted: Optional[List[str]] = None   # pod keys handed to the evictor (compared as a multiset, helper.go:299-337)
    ExpectEvictNum: Optional[int] = None
    TdmZoneActive: Optional[Dict[str, bool]] = None
    HyperNodes: Optional[List[HyperNode]] = None  # HyperNodesMap of the reference harness
    PDBs: Optional[List[PodDisruptionBudget]] = None  # what the pdb plugin lists through the informer factory

    def RegisterSession(self, tiers: Sequence[Sequence[PluginOption]], actions=("allocate",), **conf_kw) -> Snapshot:
        """conf_kw: fields of SchedulerConf, e.g. configurations={"preempt": {...}} for the reference's
        RegisterSession(tiers, []conf.Configuration)."""
        self.conf = SchedulerConf(tiers=[list(t) for t in tiers], actions=tuple(actions), **conf_kw)
        self.snap = encode_cluster(self.Nodes, self.Pods, self.PodGroups, self.Queues, self.conf,
                                   tdm_zone_active=self.TdmZoneActive, hypernodes=self.HyperNodes, pdbs=self.PDBs)
        return self.snap

    def Run(self, engine) -> AllocateResult:
        """`engine`: a Snapshot -> AllocateResult callable, or a list of Action objects like the reference's
        test.Run(actions) (uthelper/helper.go:225-236)."""
        if isinstance(engine, (list, tuple)):
            from .action import Session
            ssn = Session(self.snap)
            try:
                for act in engine:
                    act.Initialize()
                    act.Execute(ssn)
                    act.UnInitialize()
            finally:
                ssn.close()
            self.result = ssn.result
        else:
            self.result = engine(self.snap)
        # FakeBinder: Statement.Commit -> cache.AddBindTask for every Allocate op (statement.go:309-325)
        self.binds: Dict[str, str] = {}
        self.pipelined: Dict[str, List[str]] = {}
        dec, vis = self.result.decisions, self.result.visits
        for v in vis:
            ops = dec[v["first_op"]: v["first_op"] + v["n_ops"]]
            for op in ops:
                key = self.snap.task_keys[op["task"]]
                node = self.snap.node_names[op["node"]]
                if op["kind"] == abi.VC_OP_ALLOCATE and v["outcome"] == abi.VC_VISIT_COMMIT:
                    self.binds[key] = node
                elif op["kind"] == abi.VC_OP_PIPELINE:
                    self.pipelined.setdefault(self.snap.job_names[v["job"]], []).append(node)
        # FakeEvictor: Statement.Commit -> cache.Evict for every Evict op of a committed statement (statement.go:384-412)
        self.evicts: List[str] = []
        for name in ("preempt", "reclaim"):
            ar = getattr(self.result, name, None)
            if ar is None:
                continue
            for v in ar.visits:
                if v["outcome"] != abi.VC_VISIT_COMMIT:
                    continue
                for op in ar.decisions[v["first_op"]: v["first_op"] + v["n_ops"]]:
                    if op["kind"] == abi.VC_OP_EVICT:
                        self.evicts.append(self.snap.running_task_keys[op["task"]])
                    elif op["kind"] == abi.VC_OP_PIPELINE:
                        self.pipelined.setdefault(self.snap.job_names[v["job"]], []).append(self.snap.node_names[op["node"]])
        bf = getattr(self.result, "backfill", None)
        if bf is not None:  # Session.Allocate dispatches when ssn.JobReady holds (framework/session.go:785-793)
            for v in bf.visits:
                if v["outcome"] != abi.VC_VISIT_COMMIT:
                    continue
                for op in bf.decisions[v["first_op"]: v["first_op"] + v["n_ops"]]:
                    self.binds[self.snap.backfill_task_keys[op["task"]]] = self.snap.node_names[op["node"]]
        return self.result

    def CheckBind(self) -> Optional[str]:
        if self.ExpectBindsNum is not None and len(self.binds) != self.ExpectBindsNum:
            return f"case {self.Name!r}: expected {self.ExpectBindsNum} binds, got {len(self.binds)}: {self.binds}"
        if self.binds != dict(self.ExpectBindMap):
            return f"case {self.Name!r}: expected bind map {self.ExpectBindMap}, got {self.binds}"
        return None

    def CheckPipelined(self) -> Optional[str]:
        if self.ExpectPipeLined is None:
            return None
        got = {k: sorted(v) for k, v in self.pipelined.items()}
        want = {k: sorted(v) for k, v in self.ExpectPipeLined.items()}
        if got != want:
            return f"case {self.Name!r}: expected pipelined {want}, got {got}"
        return None

    def CheckEvict(self) -> Optional[str]:
        if self.ExpectEvictNum is None and self.ExpectEvicted is None:
            return None
        want = sorted(self.ExpectEvicted or [])
        if self.ExpectEvictNum is not None and self.ExpectEvictNum != len(want):
            return f"case {self.Name!r}: invalid setting: ExpectEvictNum {self.ExpectEvictNum} vs {want}"
        if sorted(self.evicts) != want:
            return f"case {self.Name!r}: expected evictions {want}, got {sorted(self.evicts)}"
        return None

    def CheckAll(self) -> Optional[str]:
        return self.CheckBind() or self.CheckEvict() or self.CheckPipelined()
