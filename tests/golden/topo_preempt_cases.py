"""actions/preempt/preempt_test.go:427-747 TestTopologyAwarePreempt, 9 of its 12 cases, with the reference's tiers
(:705-735). Left out: the two whose preemptor or victim is a BestEffort pod (vc_preempt_run refuses BestEffort pending
tasks) and the PodAntiAffinity case (inter-pod affinity is not modelled). The reference's tiers also list capacity with only
EnabledQueueOrder; it is dropped here: in every kept case one queue holds all the preemptors, so queue order never decides.
Priority classes high-priority = 100000 and low-priority = 10 appear as the resolved PodGroup priority. The test runs the
preempt action alone with {"enableTopologyAwarePreemption": true}.
"""
from volcano_b200.api import (BuildNode, BuildPod, BuildPodGroup, BuildPodGroupWithPrio, BuildPodWithPreemptionPolicy,
                              BuildPodWithPriority, BuildQueue, BuildResourceList)
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct

HIGH_PRIO, LOW_PRIO = 100000, 10
PREEMPTABLE, NOT_PREEMPTABLE = {"volcano.sh/preemptable": "true"}, {"volcano.sh/preemptable": "false"}
TOPO = {"preempt": {"enableTopologyAwarePreemption": True}}


def topo_tiers(proportion_predicate: bool = True):
    """preempt_test.go:705-735 without capacity (see the module docstring)."""
    return [[
        PluginOption.make("conformance", EnabledPreemptable=True),
        PluginOption.make("gang", EnabledPreemptable=True, EnabledJobPipelined=True, EnabledJobStarving=True),
        PluginOption.make("priority", EnabledTaskOrder=True, EnabledJobOrder=True, EnabledPreemptable=True,
                          EnabledJobPipelined=True, EnabledJobStarving=True),
        PluginOption.make("proportion", EnabledOverused=True, EnabledAllocatable=True, EnabledQueueOrder=True,
                          EnabledPredicate=proportion_predicate),
        PluginOption.make("predicates", EnabledPreemptable=True, EnabledPredicate=True),
    ]]


def _node(name, cpu, mem, pods="10"):
    return BuildNode(name, BuildResourceList(cpu, mem, ("pods", pods)))


def _queue_prio(name, priority, cap):
    """util.BuildQueueWithPriorityAndResourcesQuantity(name, priority, deserved, cap): Spec.Deserved is read by capacity
    only, which these tiers do not load."""
    q = BuildQueue(name, 1, cap)
    q.priority = priority
    return q


def golden_cases():
    """The 9 kept cases of TestTopologyAwarePreempt with their expected evictions."""
    R1 = BuildResourceList("1", "1G")
    return [
        TestCommonStruct(
            Name="do not preempt if there are enough idle resources",
            PodGroups=[BuildPodGroup("pg1", "c1", "q1", 3, {"": 3}, "Inqueue")],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", R1, "pg1"),
                  BuildPod("c1", "preemptee2", "n1", "Running", R1, "pg1"),
                  BuildPod("c1", "preemptor1", "", "Pending", R1, "pg1")],
            Nodes=[_node("n1", "10", "10G")], Queues=[BuildQueue("q1", 1, None)], ExpectEvictNum=0),
        TestCommonStruct(
            Name="do not preempt if job is pipelined",
            PodGroups=[BuildPodGroup("pg1", "c1", "q1", 1, {"": 2}, "Inqueue"), BuildPodGroup("pg2", "c1", "q1", 1, {"": 2}, "Inqueue")],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", R1, "pg1"),
                  BuildPod("c1", "preemptee2", "n1", "Running", R1, "pg1"),
                  BuildPod("c1", "preemptee3", "n1", "Running", R1, "pg2"),
                  BuildPod("c1", "preemptor2", "", "Pending", R1, "pg2")],
            Nodes=[_node("n1", "3", "3G")], Queues=[BuildQueue("q1", 1, None)], ExpectEvictNum=0),
        TestCommonStruct(
            Name="preempt one task of different job to fit both jobs on one node",
            PodGroups=[BuildPodGroupWithPrio("pg1", "c1", "q1", 1, {"": 2}, "Inqueue", LOW_PRIO),
                       BuildPodGroupWithPrio("pg2", "c1", "q1", 1, {"": 2}, "Inqueue", HIGH_PRIO)],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", R1, "pg1", PREEMPTABLE),
                  BuildPod("c1", "preemptee2", "n1", "Running", R1, "pg1", NOT_PREEMPTABLE),
                  BuildPod("c1", "preemptor1", "", "Pending", R1, "pg2"),
                  BuildPod("c1", "preemptor2", "", "Pending", R1, "pg2")],
            Nodes=[_node("n1", "2", "2G")], Queues=[BuildQueue("q1", 1, None)],
            ExpectEvicted=["c1/preemptee1"], ExpectEvictNum=1),
        TestCommonStruct(
            Name="preempt enough tasks to fit large task of different job",
            PodGroups=[BuildPodGroupWithPrio("pg1", "c1", "q1", 1, {"": 3}, "Inqueue", LOW_PRIO),
                       BuildPodGroupWithPrio("pg2", "c1", "q1", 1, {"": 1}, "Inqueue", HIGH_PRIO)],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", R1, "pg1", PREEMPTABLE),
                  BuildPod("c1", "preemptee2", "n1", "Running", R1, "pg1", PREEMPTABLE),
                  BuildPod("c1", "preemptee3", "n1", "Running", R1, "pg1", NOT_PREEMPTABLE),
                  BuildPod("c1", "preemptor1", "", "Pending", BuildResourceList("5", "5G"), "pg2")],
            Nodes=[_node("n1", "6", "6G")], Queues=[BuildQueue("q1", 1, None)],
            ExpectEvicted=["c1/preemptee2", "c1/preemptee1"], ExpectEvictNum=2),
        TestCommonStruct(  # issue #3161
            Name="preempt low priority job in same queue",
            PodGroups=[BuildPodGroupWithPrio("pg1", "c1", "q1", 0, {}, "Inqueue", LOW_PRIO),
                       BuildPodGroupWithPrio("pg2", "c1", "q1", 1, {"": 1}, "Inqueue", HIGH_PRIO)],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", BuildResourceList("3", "3G"), "pg1", PREEMPTABLE),
                  BuildPod("c1", "preemptor1", "", "Pending", BuildResourceList("3", "3G"), "pg2")],
            Nodes=[_node("n1", "12", "12G")], Queues=[BuildQueue("q1", 1, BuildResourceList("4", "4G"))],
            ExpectEvicted=["c1/preemptee1"], ExpectEvictNum=1),
        TestCommonStruct(
            Name="preempt low priority job in same queue: allocatable and has enough resource, don't preempt",
            PodGroups=[BuildPodGroupWithPrio("pg1", "c1", "q1", 1, {}, "Inqueue", LOW_PRIO),
                       BuildPodGroupWithPrio("pg2", "c1", "q1", 1, {"": 1}, "Inqueue", HIGH_PRIO)],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", BuildResourceList("3", "3G"), "pg1", PREEMPTABLE),
                  BuildPod("c1", "preemptor1", "", "Pending", BuildResourceList("3", "3G"), "pg2")],
            Nodes=[_node("n1", "12", "12G")], Queues=[BuildQueue("q1", 1, BuildResourceList("6", "6G"))],
            ExpectEvictNum=0),
        TestCommonStruct(  # issue #2232
            Name="preempt low priority job in same queue but not pod with preemptable=false or higher priority",
            PodGroups=[BuildPodGroupWithPrio("pg1", "c1", "q1", 1, {}, "Inqueue", LOW_PRIO),
                       BuildPodGroupWithPrio("pg2", "c1", "q1", 1, {"": 1}, "Inqueue", HIGH_PRIO)],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", R1, "pg1", NOT_PREEMPTABLE),
                  BuildPod("c1", "preemptee2", "n1", "Running", R1, "pg1", PREEMPTABLE),
                  BuildPodWithPriority("c1", "preemptee3", "n1", "Running", R1, "pg1", PREEMPTABLE, None, HIGH_PRIO),
                  BuildPod("c1", "preemptor1", "", "Pending", R1, "pg2")],
            Nodes=[_node("n1", "12", "12G")], Queues=[BuildQueue("q1", 1, BuildResourceList("3", "3G"))],
            ExpectEvicted=["c1/preemptee2"], ExpectEvictNum=1),
        TestCommonStruct(  # issue #3642
            Name="can not preempt resources when task preemption policy is never",
            PodGroups=[BuildPodGroupWithPrio("pg1", "c1", "q1", 0, None, "Inqueue", LOW_PRIO),
                       BuildPodGroupWithPrio("pg2", "c1", "q1", 1, None, "Inqueue", HIGH_PRIO)],
            Pods=[BuildPod("c1", "preemptee1", "n1", "Running", R1, "pg1", PREEMPTABLE),
                  BuildPodWithPreemptionPolicy("c1", "preemptor1", "", "Pending", R1, "pg2", None, None, "Never")],
            Nodes=[_node("n1", "1", "1Gi", "1")], Queues=[BuildQueue("q1", 1, None)],
            ExpectEvicted=[], ExpectEvictNum=0),
        TestCommonStruct(
            Name="preemption with priority queues",
            PodGroups=[BuildPodGroupWithPrio("pg3", "c1", "q2", 1, None, "Running", HIGH_PRIO),
                       BuildPodGroupWithPrio("pg1", "c1", "q1", 0, None, "Running", LOW_PRIO),
                       BuildPodGroupWithPrio("pg2", "c1", "q1", 1, None, "Inqueue", HIGH_PRIO)],
            Pods=[BuildPod("c1", "preemptee2", "n1", "Running", R1, "pg3", PREEMPTABLE),
                  BuildPod("c1", "preemptee1", "n1", "Running", R1, "pg1", PREEMPTABLE),
                  BuildPodWithPreemptionPolicy("c1", "preemptor1", "", "Pending", R1, "pg2", None, None, "PreemptLowerPriority")],
            Nodes=[_node("n1", "2", "2Gi", "2")],
            Queues=[_queue_prio("q1", 1, BuildResourceList("1", "1G")), _queue_prio("q2", 10, BuildResourceList("1", "1G"))],
            ExpectEvicted=["c1/preemptee1"], ExpectEvictNum=1),
    ]
