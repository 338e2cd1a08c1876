"""The pdb and cdp victim votes on the CPU: the reference's plugin tests transcribed onto the guard oracle's votes and the
session encoder, and the hand-derived action-level sessions of tests/guard_cases.py on the oracle."""
import pytest

from tests import guard_cases as GC
from tests import guard_common as G
from volcano_b200 import abi
from volcano_b200.api import BuildNode, BuildPDB, BuildPod, BuildPodGroup, BuildQueue, BuildResourceList, go_parse_duration
from volcano_b200.snapshot import PluginOption
from volcano_b200.uthelper import TestCommonStruct

LABEL = "volcano.sh/job-name"


def _vote_session(pods, pdbs, plugin, now=0):
    tc = TestCommonStruct(Name="vote")
    tc.Nodes = [BuildNode("n0", BuildResourceList("8", "8G", ("pods", "10")))]
    tc.Queues = [BuildQueue("q", 1)]
    tc.PodGroups = [BuildPodGroup("pg", "default", "q", 1)]
    tc.Pods = pods
    tc.PDBs = pdbs
    return tc.RegisterSession([[PluginOption.make(plugin, EnabledPreemptable=True, EnabledReclaimable=True)]],
                              actions=("preempt",), now_ns=now)


@pytest.mark.parametrize("pdbs,want", [
    ([], [0, 1]),                                                   # "test without pdbs"
    ([BuildPDB("default", "test-pdb", {LABEL: "job-1"}, 0)], []),   # "test with pdbs(can evict 0 pod)"
    ([BuildPDB("default", "test-pdb", {LABEL: "job-1"}, 1)], [0]),  # "test with pdbs(can evict 1 pod)"
])
def test_pdb_preemptable_and_reclaimable_fn(pdbs, want):
    """plugins/pdb/pdb_test.go TestPreemptableAndReclaimableFn: test-pod1 and test-pod2 (label volcano.sh/job-name=job-1,
    namespace default) against no PDB, a PDB allowing 0 and one allowing 1."""
    pods = [BuildPod("default", f"test-pod{i + 1}", "n0", "Running", BuildResourceList("1", "1G"), "pg", {LABEL: "job-1"})
            for i in range(2)]
    snap = _vote_session(pods, pdbs, "pdb")
    o = G.GuardOracle(snap)
    try:
        assert o.vote(abi.VC_PLUGIN_PDB, [0, 1]) == want
    finally:
        o.close()


def test_cdp_pod_cooldown_time():
    """plugins/cdp/cdp_test.go Test_CooldownTimePlugin_podPreemptStableTime: "600s" is enabled with 600 s, "600abcde" is
    not; the encoder parses durations as time.ParseDuration does."""
    assert go_parse_duration("600s") == 600 * 10 ** 9
    assert go_parse_duration("600abcde") is None
    assert go_parse_duration("1h2m3.5s") == (3723 * 10 ** 9 + 5 * 10 ** 8)
    assert go_parse_duration("0") == 0 and go_parse_duration("") is None and go_parse_duration("10") is None


def test_cdp_preemptable_fn():
    """plugins/cdp/cdp_test.go TestPreemptableFn: task1 (600s, scheduled 100 s ago) is kept, task2 (invalid "600abcde") and
    task3 (600s, scheduled 800 s ago) are victims."""
    now = 10 ** 18
    pods = []
    for name, cool, ago in (("t1", "600s", 100), ("t2", "600abcde", 100), ("t3", "600s", 800)):
        p = BuildPod("default", name, "n0", "Running", BuildResourceList("1", "1G"), "pg", {"volcano.sh/preemptable": "true"})
        p.annotations = {"volcano.sh/cooldown-time": cool}
        p.scheduled_time = now - ago * 10 ** 9
        pods.append(p)
    snap = _vote_session(pods, [], "cdp", now)
    assert list(snap.g_until) == [now + 500 * 10 ** 9, abi.VC_COOLDOWN_NONE, now - 200 * 10 ** 9]
    o = G.GuardOracle(snap)
    try:
        assert o.vote(abi.VC_PLUGIN_CDP, [0, 1, 2]) == [1, 2]
    finally:
        o.close()


def test_invalid_label_disables_valid_annotation():
    """cdp.go:58-70: the label is read first; an unparsable label disables cooldown even when the annotation parses."""
    p = BuildPod("default", "t", "n0", "Running", BuildResourceList("1", "1G"), "pg", {"volcano.sh/cooldown-time": "x"})
    p.annotations = {"volcano.sh/cooldown-time": "600s"}
    p.scheduled_time = 0
    snap = _vote_session([p], [], "cdp", 1)
    assert snap.g_until[0] == abi.VC_COOLDOWN_NONE


def test_encoder_pdb_table():
    """The encoder's table: per running task the PDBs that count it (namespace, matchLabels, DisruptedPods), the
    no-labels flag, DisruptionsAllowed per PDB; an empty selector counts nothing."""
    mk = lambda name, ns, labels: BuildPod(ns, name, "n0", "Running", BuildResourceList("1", "1G"), "pg", labels)
    pods = [mk("a", "default", {"app": "x", "tier": "1"}), mk("b", "default", {}), mk("c", "other", {"app": "x"}),
            mk("d", "default", {"app": "x"})]
    pdbs = [BuildPDB("default", "p0", {"app": "x"}, 2, ["d"]), BuildPDB("default", "p1", {"tier": "1"}, 0),
            BuildPDB("default", "p2", {}, 5), BuildPDB("other", "p3", {"app": "x"}, 1)]
    snap = _vote_session(pods, pdbs, "pdb")
    rows = [list(snap.g_pdb[snap.g_pdb_off[r]:snap.g_pdb_off[r + 1]]) for r in range(4)]
    assert rows == [[0, 1], [], [3], []]
    assert list(snap.g_flags) == [0, abi.VC_GUARD_NO_LABELS, 0, 0]
    assert list(snap.g_pdb_allowed) == [2, 0, 5, 1]


@pytest.mark.parametrize("case", sorted(GC.CASES))
def test_hand_derived_cases_on_the_oracle(case):
    snap, want = GC.CASES[case]()
    assert sorted(G.evicted(snap, G.run(snap))) == want


def test_oracle_refuses_votes_without_a_table():
    snap, _ = GC.budget_one_two_pods()
    snap.g_pdb_off = None  # no table
    with pytest.raises(RuntimeError, match="rc=-1"):
        G.run(snap)


def test_restated_actions_match_the_sampling_oracle_without_guards():
    """With pdb and cdp out of the tiers the guard oracle's restated actions give the sampling oracle's statements."""
    from tools.fuzz_evict import make_guard_case
    from tests import samp_common as S
    checked = 0
    for seed in range(200):
        tc, tiers, actions, conf = make_guard_case(seed)
        bare = [[o for o in t if o.name not in ("pdb", "cdp")] for t in tiers]
        snap = tc.RegisterSession(bare, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        assert S.same(G.run(snap), S.run(snap)), seed
        checked += 1
    assert checked >= 150
