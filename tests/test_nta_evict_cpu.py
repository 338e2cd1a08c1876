"""Preempt and reclaim with the network-topology-aware plugin on the CPU: the hand-derived sessions of
tests/nta_cases.py on the oracle extension (tools/nta_evict_oracle), the plugin's cache after each action, and the
extension against the guard oracle on sessions without the plugin or topology jobs."""
import pytest

from tests import guard_common as G
from tests import nta_cases as NC
from tests import nta_common as N
from tests import samp_common as S


@pytest.mark.parametrize("case", sorted(NC.CASES))
def test_hand_derived_cases(case):
    snap, want = NC.CASES[case]()
    assert sorted(G.evicted(snap, N.run(snap))) == want


def test_without_the_plugin_the_first_node_wins():
    snap, want = NC.term_changes_the_node(nta=False)
    assert sorted(G.evicted(snap, N.run(snap))) == want == ["ns/r0"]


def test_discard_books_only_committed_statements():
    """After big's discarded statement, hyperNodeResourceCache.used moves only by the committed statements: on hnB, r1 out
    and two pods of 4 cpus / 1G in (small's, then in the intra-job phase one of big's, pipelined into the 4 cpus n1 has
    left with no victim); hnA keeps its opening value."""
    snap, _ = NC.discard_restores_used()
    keep = []
    N.run(snap, keep)
    used = keep[-1][1]
    cpu, mem = 1000.0, 1e9  # the encoder's units: millicores, bytes
    hn = {name: i for i, name in enumerate(snap.hn_names)}
    assert used[hn["hnA"]][:2].tolist() == [12 * cpu, 4 * mem]
    assert used[hn["hnB"]][:2].tolist() == [(12 - 6 + 4 + 4) * cpu, (32 - 16 + 1 + 1) * mem]


def test_reclaim_books_the_cache_for_preempt():
    snap, _ = NC.reclaim_then_preempt()
    keep = []
    N.run(snap, keep)
    hn = {name: i for i, name in enumerate(snap.hn_names)}
    assert keep[0][0] == "reclaim"
    assert keep[0][1][hn["hnA"]][:2].tolist() == [12 * 1000.0, 33 * 1e9]


def test_without_the_plugin_the_guard_oracle_statements():
    """Sessions of make_guard_case (no network-topology-aware plugin, no topology job): the extension's preempt and
    reclaim give the guard oracle's statements, visits and indexes."""
    from tools.fuzz_evict import make_guard_case
    ran = 0
    for seed in range(80):
        tc, tiers, actions, conf = make_guard_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        assert S.same(N.run(snap), G.run(snap)), seed
        ran += 1
    assert ran >= 60


def test_family_sessions_run_on_the_oracle():
    """make_nta_case sessions run on the extension, and the plugin changes preempt / reclaim statements in some of them
    that start from the same allocate placements."""
    from tools.fuzz_evict import make_nta_case, without_nta
    changed = evictions = 0
    for seed in range(360):
        tc, tiers, actions, conf = make_nta_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = N.run(snap)
        evictions += len(G.evicted(snap, ref))
        changed += N.evict_changed(ref, N.run(tc.RegisterSession(without_nta(tiers), actions=actions, **conf)))
    assert evictions > 0 and changed >= 10, (evictions, changed)


def test_tdm_stays_refused():
    snap = NC.with_tdm()
    o = N.NtaOracle(snap)
    try:
        with pytest.raises(RuntimeError, match="rc=-4"):
            o.preempt()
    finally:
        o.close()
