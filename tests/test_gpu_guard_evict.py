"""Preempt and reclaim with the pdb and cdp plugins on the H100:
- the hand-derived sessions of tests/guard_cases.py give their derived evictions through the library;
- random sessions of tools/fuzz_evict.make_guard_case (normal and topology-aware readings, with and without sampling)
  give the guard oracle's statements exactly, and the family contains sessions where the guards change them;
- a session where pdb or cdp votes and no table is set is refused with VC_EINVAL;
- allocate and backfill give the same results with and without the two plugins in the tiers."""
import numpy as np
import pytest

from tests import guard_cases as GC
from tests import guard_common as G
from tests import samp_common as S
from volcano_b200 import abi

pytestmark = pytest.mark.gpu


def _gpu(snap):
    from volcano_b200 import engine
    engine.init(0)
    return engine.gpu_engine(snap)


@pytest.mark.parametrize("case", sorted(GC.CASES))
def test_hand_derived_cases(case):
    snap, want = GC.CASES[case]()
    assert sorted(G.evicted(snap, _gpu(snap))) == want


def test_votes_without_a_table_are_refused():
    from volcano_b200 import engine
    snap, _ = GC.budget_one_two_pods()
    snap.g_pdb_off = None
    with pytest.raises(engine.VcError) as ei:
        _gpu(snap)
    assert ei.value.code == abi.VC_EINVAL


def _without_guards(tiers):
    return [[o for o in t if o.name not in ("pdb", "cdp")] for t in tiers]


def test_sessions_match_the_oracle():
    """400 random sessions of make_guard_case: allocate placements, preempt / reclaim statements and visits, and under
    sampling the index, identical to the guard oracle. Not vacuous: the oracle's statements change without pdb and cdp in
    sessions of both readings."""
    from tools.fuzz_evict import make_guard_case
    checked, evictions = 0, 0
    changed = {"normal": 0, "topo": 0}
    for seed in range(400):
        tc, tiers, actions, conf = make_guard_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = G.run(snap)
        res = _gpu(snap)
        assert S.same(res, ref), (seed, actions, conf)
        checked += 1
        evictions += len(G.evicted(snap, ref))
        bare = G.run(tc.RegisterSession(_without_guards(tiers), actions=actions, **conf))
        if not S.same(ref, bare, index=False):
            changed["topo" if "configurations" in conf else "normal"] += 1
    assert checked >= 300 and evictions > 0
    assert changed["normal"] >= 5 and changed["topo"] >= 3, changed


def test_allocate_and_backfill_ignore_the_guards():
    """The two plugins register no allocate-path function: make_case clusters run allocate and backfill to the same
    decisions with pdb and cdp in the tiers and without."""
    from tools.fuzz_evict import make_case
    from volcano_b200.snapshot import PluginOption
    ran = 0
    for seed in range(60):
        tc, tiers, _ = make_case(seed)
        plain = tc.RegisterSession(tiers, actions=("allocate", "backfill"))
        if plain.T + plain.B == 0 or plain.N == 0:
            continue
        a = _gpu(plain)
        guarded = [list(t) for t in tiers]
        guarded[0] = guarded[0] + [PluginOption.defaults("pdb"), PluginOption.defaults("cdp")]
        b = _gpu(tc.RegisterSession(guarded, actions=("allocate", "backfill")))
        assert np.array_equal(a.decisions, b.decisions) and np.array_equal(a.visits, b.visits), seed
        if a.backfill is not None or b.backfill is not None:
            assert np.array_equal(a.backfill.decisions, b.backfill.decisions), seed
        ran += 1
    assert ran >= 40
