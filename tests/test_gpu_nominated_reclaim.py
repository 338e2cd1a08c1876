"""Reclaim on sessions with nominated pending pods on the H100: the hand-derived case of tests/nominated_cases.py, random
sessions of tools/fuzz_evict.make_case with NominatedNodeName on about half the pending pods (allocate -> reclaim and
reclaim alone) against the oracle statement by statement, and preempt's refusal of such sessions."""
import pytest

from tests import nominated_cases as NC
from tests import samp_cases as SC

pytestmark = pytest.mark.gpu


def _engine():
    from volcano_b200 import engine
    engine.init(0)
    return engine


@pytest.mark.parametrize("nominated", ["n0", "gone"])
@pytest.mark.parametrize("actions", [("reclaim",), ("allocate", "reclaim")])
def test_hand_derived_case(nominated, actions):
    snap, want = NC.reclaim_case(nominated, actions)
    assert SC.statements(snap, _engine().gpu_engine(snap).reclaim) == want


def test_random_sessions_match_the_oracle(oracle_engine):
    """Not vacuous: sessions where a pod is nominated to a node of the session and reclaim evicts."""
    from tools import fuzz_evict as F
    engine = _engine()
    checked = with_evictions = 0
    for seed in range(400):
        tc, tiers, actions = F.make_case(seed)
        if not NC.nominate(tc, seed):
            continue
        actions = ("allocate", "reclaim") if seed % 2 else ("reclaim",)
        snap = tc.RegisterSession(tiers, actions=actions)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = oracle_engine(snap)
        res = engine.gpu_engine(snap)
        F.compare(res, ref, seed)
        checked += 1
        if (snap.t_nominated >= 0).any() and len(ref.reclaim.decisions):
            with_evictions += 1
    assert checked >= 300 and with_evictions >= 8, (checked, with_evictions)


def test_preempt_still_refuses_a_nominated_session():
    """The same session with preempt: VC_EUNSUPPORTED from vc_preempt_run, after reclaim ran on it."""
    snap, _ = NC.reclaim_case("n0", ("reclaim", "preempt"))
    engine = _engine()
    e = engine.Engine(snap)
    try:
        e.upload()
        e.reclaim()
        with pytest.raises(Exception, match="NominatedNodeName|-2|UNSUPPORTED"):
            e.preempt()
    finally:
        e.close()
