"""Hierarchical drf (drf's enableHierarchy) on the CPU: the upstream TestHDRF tables, hand-derived tree states, the queue
heap, the refusals, and the Python encoder. The oracle here is tools/hdrf_oracle (a plain restatement of drf.go over the
unchanged CPU oracle)."""
import numpy as np
import pytest

from tests import hdrf_common as H
from volcano_b200.api import BuildNode, BuildPodGroup, BuildQueueWithAnnos, BuildResourceList
from volcano_b200.snapshot import go_parse_float
from volcano_b200.uthelper import TestCommonStruct

G = 1e9


def _run(case, check=True, **kw):
    snap = case.RegisterSession(H.tiers(**kw))
    o = H.oracle_for(snap, case.Queues)
    assert o.attach_rc == 0 or not check
    return snap, o


def test_upstream_rescaling():
    """hdrf_test.go "rescaling test" (tiers: drf with hierarchy + queue / job order, proportion with queue order; proportion's
    deserved shares take part in the chain after hdrf). The code's result equals the authors' table: 5 pods each; sci gets
    (5 cpu, 5G), eng's two teams split eng's half by their dominant resource."""
    snap, o = _run(H.rescaling_case())
    al = H.per_job_allocated(snap, o.allocate()[0])
    assert np.array_equal(al["default/pg1"], [5000, 5 * G, 5])
    assert np.array_equal(al["default/pg21"], [5000, 0, 5])
    assert np.array_equal(al["default/pg22"], [0, 5 * G, 5])


def test_upstream_blocking_nodes():
    """hdrf_test.go "blocking nodes test": pg31 and pg32 share the node root/pg3/pg31. cpu runs out after pg1, pg2 and
    pg31 hold 10 cpu each; the cpu jobs' leaves are then saturated (cpu no longer demanding) and memory goes to pg32 and pg4,
    15G each. Equal to the authors' table."""
    snap, o = _run(H.blocking_case())
    al = H.per_job_allocated(snap, o.allocate()[0])
    for pg in ("pg1", "pg2", "pg31"):
        assert np.array_equal(al[f"default/{pg}"], [10000, 0, 10]), pg
    for pg in ("pg32", "pg4"):
        assert np.array_equal(al[f"default/{pg}"], [0, 15 * G, 15]), pg


def test_heap_layout_matters():
    """The queue PQ is a Go heap that is not re-sifted when a placement moves the shares of waiting queues. On the
    rescaling case, serving the arg-min of the live keys instead gives a different placement sequence: the heap is
    what makes the result exact."""
    snap, o = _run(H.rescaling_case())
    heap = o.allocate()[0]
    _, o2 = _run(H.rescaling_case())
    argmin = o2.allocate(argmin=True)[0]
    assert len(heap) == len(argmin) == 15
    assert not np.array_equal(heap["task"], argmin["task"])


def _two_level(weights=("1/2", "1/3/1", "1/3/1"), allocs=((2000, 0), (1000, 0), (0, 3)), check=True):
    """root -> {x (queue qx), y -> {y1 (qy1), y2 (qy2)}}; one job per queue with the given (cpu milli, GB) allocated."""
    from volcano_b200.api import BuildPod
    pods, pgs = [], []
    for k, (name, (cpu, mem)) in enumerate(zip(("jx", "jy1", "jy2"), allocs)):
        pgs.append(BuildPodGroup(name, "default", ("qx", "qy1", "qy2")[k], 0, None, "Inqueue"))
        pods.append(BuildPod("default", f"{name}-run", "n", "Running", BuildResourceList(f"{cpu}m", f"{mem}G"), name))
        pods.append(BuildPod("default", f"{name}-p", "", "Pending", BuildResourceList("1", "1G"), name))
    queues = [BuildQueueWithAnnos("qx", 1, None, {H.HIER: "root/x", H.WEIGHTS: weights[0]}),
              BuildQueueWithAnnos("qy1", 1, None, {H.HIER: "root/y/y1", H.WEIGHTS: weights[1]}),
              BuildQueueWithAnnos("qy2", 1, None, {H.HIER: "root/y/y2", H.WEIGHTS: weights[2]})]
    case = TestCommonStruct(Name="two-level", PodGroups=pgs, Pods=pods, Queues=queues,
                            Nodes=[BuildNode("n", BuildResourceList("10", "10G", ("pods", "100")))])
    return _run(case, check)


def test_mdr_rescaling_by_hand():
    """y's children: jy1 share 1000/10000 = 0.1 (cpu), jy2 share 3G/10G = 0.3 (memory). mdr = 0.1, so jy2 is scaled by
    0.1 / 0.3: y.allocated = (1000, 0) + (0, 3G) * (1/3) -> share max(0.1, 0.1) = 0.1 (up to the rounding of 1/3)."""
    snap, o = _two_level()
    s_y, w_y, sat_y, a_y = o.node(1, 1)
    ratio = 0.1 / 0.3
    assert a_y[0] == 1000.0 and a_y[1] == 3e9 * ratio
    assert s_y == max(1000.0 / 10000.0, 3e9 * ratio / 10e9) and w_y == 3.0 and not sat_y
    s_x, w_x, _, _ = o.node(0, 1)
    assert s_x == 0.2 and w_x == 2.0
    # x: 0.2 / 2 = 0.1 against y: ~0.1 / 3: qy1 first
    assert o.compare(1, 0) < 0 and o.compare(0, 1) > 0


def test_saturated_leaf_added_unscaled():
    """A leaf whose allocation reached its request in some dimension is saturated and enters its parent's sum as it is."""
    snap, o = _two_level()
    # jy1 requests 1000m (running) + 1 cpu (pending): give it its whole request
    o.job_add(1, [1000, 1e9, 1])
    s_y, _, sat_y, a_y = o.node(1, 1)
    # jy1 (saturated): (2000, 1G) unscaled; jy2 alone sets mdr = 0.3 and keeps its scale 1
    assert not sat_y and a_y[0] == 2000.0 and a_y[1] == 1e9 + 3e9


def test_demanding_change_saturates_other_subtrees():
    """When cpu stops being demanding (totalAllocated reaches the total), every leaf with cpu allocated and requested is
    saturated, in any subtree."""
    snap, o = _two_level()
    assert not o.node(0, 1)[2]
    o.job_add(2, [7000, 0, 0])  # 2000 + 1000 + 7000 = the cluster's 10 cpu
    assert o.node(0, 1)[2]      # x: jx has cpu allocated and requested
    assert o.node(1, 2)[2]      # y1 likewise


def test_weight_clamp():
    """"0.5" and "abc" (ParseFloat error -> 0) both become weight 1."""
    for w in ("1/0.5", "1/abc"):
        _, o = _two_level(weights=(w, "1/3/1", "1/3/1"))
        assert o.node(0, 1)[1] == 1.0


def test_first_creator_weight_wins():
    """qy1 creates y (its job has the lower index) with weight 3; qy2 names y with weight 7, which changes nothing."""
    _, o = _two_level(weights=("1/2", "1/3/1", "1/7/1"))
    assert o.node(2, 1)[1] == 3.0


def test_root_level_queue_ties():
    """A queue with an empty hierarchy sits at the root: compareQueues ends after the root level and returns 0."""
    from volcano_b200.api import BuildPod
    case = TestCommonStruct(
        Name="root", Nodes=[BuildNode("n", BuildResourceList("10", "10G", ("pods", "100")))],
        PodGroups=[BuildPodGroup("j0", "default", "q0", 0, None, "Inqueue"), BuildPodGroup("j1", "default", "q1", 0, None, "Inqueue")],
        Pods=[BuildPod("default", "j0-p", "", "Pending", BuildResourceList("1", "1G"), "j0"),
              BuildPod("default", "j1-r", "n", "Running", BuildResourceList("3", "1G"), "j1"),
              BuildPod("default", "j1-p", "", "Pending", BuildResourceList("1", "1G"), "j1")],
        Queues=[BuildQueueWithAnnos("q0", 1, None, {}), BuildQueueWithAnnos("q1", 1, None, {H.HIER: "root/a", H.WEIGHTS: "1/1"})])
    snap, o = _run(case)
    assert o.compare(0, 1) == 0 and o.compare(1, 0) == 0


def test_refusals():
    """Inputs the reference crashes on are refused: weights shorter than the path, and a job whose queue is not in the
    session."""
    _, o = _two_level(weights=("1/2", "1/3", "1/3/1"), check=False)
    assert o.attach_rc != 0
    from volcano_b200.api import BuildPod
    case = TestCommonStruct(
        Name="orphan", Nodes=[BuildNode("n", BuildResourceList("10", "10G", ("pods", "100")))],
        PodGroups=[BuildPodGroup("j0", "default", "missing", 0, None, "Inqueue")],
        Pods=[BuildPod("default", "j0-p", "", "Pending", BuildResourceList("1", "1G"), "j0")],
        Queues=[BuildQueueWithAnnos("q0", 1, None, {H.HIER: "root/a", H.WEIGHTS: "1/1"})])
    snap = case.RegisterSession(H.tiers())
    assert H.oracle_for(snap, case.Queues).attach_rc != 0


def test_encoder():
    """The table the Python encoder builds: segments below the root, interned names, ParseFloat values."""
    assert go_parse_float("2.5") == 2.5 and go_parse_float("abc") == 0.0 and go_parse_float("1e400") == float("inf")
    assert go_parse_float(" 2") == 0.0 and go_parse_float("1_0") == 0.0 and go_parse_float("+nan") == 0.0
    # hexadecimal mantissa with a p exponent, underscores only after a base prefix
    assert go_parse_float("0x10p0") == 16.0 and go_parse_float("0x1_0p0") == 16.0 and go_parse_float("0x_10p0") == 16.0
    assert go_parse_float("0x10") == 0.0 and go_parse_float("0x1__0p0") == 0.0
    snap, _ = _two_level(weights=("1/2", "1/3/1", "1/7/x"))
    assert snap.hd_path_off.tolist() == [0, 1, 3, 5]
    assert snap.hd_path_name.tolist() == [0, 1, 2, 1, 3]
    assert snap.hd_weight.tolist() == [2.0, 3.0, 1.0, 7.0, 0.0]
    assert snap.hd_n_weights.tolist() == [1, 2, 2]
    # TotalRequest: the running pod and the pending one
    assert snap.hd_job_request[:, 0].tolist() == [3000, 1e9, 2]
