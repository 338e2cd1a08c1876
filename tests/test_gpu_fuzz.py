"""Randomised differential parity: API-level clusters (tools/fuzz_api.py generator: labels, affinity, taints of every
effect, tolerations, tdm zones, running / deleting pods, roles, queue caps and priorities, HyperNode trees with
soft-mode topology jobs, random plugin sets and arguments) — CUDA path vs CPU oracle, bit-equal."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _generator():
    spec = importlib.util.spec_from_file_location("fuzz_api", os.path.join(ROOT, "tools", "fuzz_api.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("block", range(6))
def test_random_clusters_match_oracle(block, oracle_engine):
    from volcano_b200 import engine
    engine.init(0)
    gen = _generator()
    make_case = gen.make_case
    checked = backfilled = 0
    for seed in range(1000 + 40 * block, 1000 + 40 * (block + 1)):
        tc, tiers, actions = make_case(seed)
        if not tiers:
            continue
        if not gen.backfill_supported(tiers, tc.conf_kw):
            actions = tuple(a for a in actions if a != "backfill")
        snap = tc.RegisterSession(tiers, actions=actions, **tc.conf_kw)
        if snap.T == 0 or snap.N == 0:
            continue
        ref = oracle_engine(snap)
        res = engine.gpu_engine(snap)
        assert (res.backfill is None) == (ref.backfill is None), seed
        if ref.backfill is not None:  # the backfill action on the state allocate left
            assert np.array_equal(res.backfill.decisions, ref.backfill.decisions), seed
            assert np.array_equal(res.backfill.visits, ref.backfill.visits), seed
            assert np.array_equal(res.backfill.fit_errors, ref.backfill.fit_errors), seed
            backfilled += len(ref.backfill.decisions)
        assert np.array_equal(res.decisions, ref.decisions), seed  # tasks, nodes, kinds, visits AND fp64 scores bit-equal
        assert np.array_equal(res.visits, ref.visits), seed
        assert np.array_equal(res.fit_errors, ref.fit_errors), seed
        if ref.job_allocated_hypernodes is not None:
            assert np.array_equal(res.job_allocated_hypernodes, ref.job_allocated_hypernodes), seed
        checked += 1
    assert checked >= 30


@pytest.mark.parametrize("block", range(6))
def test_random_preempt_reclaim_match_oracle(block, oracle_engine):
    """The preempt and reclaim actions (alone, after allocate, in either order) on random clusters of running and pending
    pods (tools/fuzz_evict.py): every statement (evictions, pipelines, commit / discard) identical to the oracle's.
    Blocks 0-3: small clusters of 1-6 nodes; blocks 4-5: wide clusters (up to 3 000 mostly identical nodes, nodes running
    more than 16 pods, R > 8)."""
    from volcano_b200 import engine
    engine.init(0)
    spec = importlib.util.spec_from_file_location("fuzz_evict", os.path.join(ROOT, "tools", "fuzz_evict.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    if block < 4:
        seeds, make_case, need = range(3000 + 60 * block, 3000 + 60 * (block + 1)), gen.make_case, 40
    else:
        seeds, make_case, need = range(5000 + 20 * (block - 4), 5000 + 20 * (block - 3)), gen.make_wide_case, 20
    checked = ops = 0
    for seed in seeds:
        tc, tiers, actions = make_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        ref = oracle_engine(snap)
        res = engine.gpu_engine(snap)
        ops += gen.compare(res, ref, seed)
        checked += 1
    assert checked >= need and ops >= 1
