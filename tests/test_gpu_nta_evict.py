"""Preempt and reclaim with the network-topology-aware plugin on the H100:
- the hand-derived sessions of tests/nta_cases.py give their derived evictions through the library;
- random sessions of tools/fuzz_evict.make_nta_case (pdb / cdp, PreferNoSchedule taints, the topology-aware reading,
  sampling, soft-mode topology jobs) give the oracle extension's statements exactly, and the plugin changes the
  statements of some of them;
- a session with the tdm plugin is still refused with VC_EUNSUPPORTED."""
import pytest

from tests import guard_common as G
from tests import nta_cases as NC
from tests import nta_common as N
from tests import samp_common as S
from volcano_b200 import abi

pytestmark = pytest.mark.gpu


def _gpu(snap):
    from volcano_b200 import engine
    engine.init(0)
    return engine.gpu_engine(snap)


@pytest.mark.parametrize("case", sorted(NC.CASES))
def test_hand_derived_cases(case):
    snap, want = NC.CASES[case]()
    res = _gpu(snap)
    assert sorted(G.evicted(snap, res)) == want
    assert S.same(res, N.run(snap))


def test_tdm_is_refused():
    from volcano_b200 import engine
    with pytest.raises(engine.VcError) as ei:
        _gpu(NC.with_tdm())
    assert ei.value.code == abi.VC_EUNSUPPORTED


def test_sessions_match_the_oracle():
    """360 random sessions of make_nta_case: allocate placements, preempt / reclaim statements and visits, and under
    sampling the index, identical to the oracle. Not vacuous: without the plugin the oracle's preempt / reclaim statements
    change in some sessions whose allocate placements stay the same."""
    from tools.fuzz_evict import make_nta_case, without_nta
    checked = evictions = changed = 0
    for seed in range(360):
        tc, tiers, actions, conf = make_nta_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = N.run(snap)
        res = _gpu(snap)
        assert S.same(res, ref), (seed, actions, conf)
        checked += 1
        evictions += len(G.evicted(snap, ref))
        changed += N.evict_changed(ref, N.run(tc.RegisterSession(without_nta(tiers), actions=actions, **conf)))
    assert checked >= 300 and evictions > 0
    assert changed >= 10, changed
