"""Reclaim with a nominated pending pod on the CPU oracle: the derived statements of tests/nominated_cases.py, whether the
name is a node of the session or not, alone and after allocate."""
import pytest

from tests import nominated_cases as NC
from tests import samp_cases as SC


@pytest.mark.parametrize("nominated", ["n0", "gone"])
@pytest.mark.parametrize("actions", [("reclaim",), ("allocate", "reclaim")])
def test_oracle_gives_the_derived_statements(oracle_engine, nominated, actions):
    snap, want = NC.reclaim_case(nominated, actions)
    assert (snap.t_nominated >= 0).any() == (nominated == "n0")
    assert SC.statements(snap, oracle_engine(snap).reclaim) == want
