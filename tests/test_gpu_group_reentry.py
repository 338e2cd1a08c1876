"""Re-entry of a (class, request) group in the incremental commit kernel (k_commit_fast) from its saved verdicts.

When the kernel comes back to a group whose verdicts it saved earlier in the cycle, it takes them from the per-group
verdict table and re-evaluates only the rows that changed since. Every case runs against the CPU oracle's allocate()
on the same session: decisions (task, node, kind, visit, fp64 score), visits and fit errors are bit-equal. With VC_PROF,
vc_stats.group_reentry says which path each group switch took:
  [0] switches served by a full sweep, [1] served from the table (control program: the same on every CTA),
  [2] rows re-evaluated on re-entry, [3] CTA re-entries past the changed-row threshold (summed over CTAs);
and [0] + [1] is the number of steps that swept (prof_cycles[6]). Each case asserts the path it is there to take."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

VT_BUDGET = 256 << 20  # kVerdictTableBudget: n_groups x node slots x 9 B above it keeps full sweeps


@pytest.fixture(scope="module")
def gpu():
    from volcano_b200 import engine
    engine.init(0)
    return engine


def _snap(base, **changes):
    from volcano_b200.synth import CONFIGS, make_snapshot
    cfg = dataclasses.replace(CONFIGS[base], name=f"{base}-reentry", **changes)
    return make_snapshot(cfg)


def _run(gpu, snap, opts=None, cycles=1):
    opts = dict(opts or {}, VC_PROF=1)
    for k, v in opts.items():
        gpu.debug_option(k, v)
    try:
        e = gpu.Engine(snap)
        out = []
        for _ in range(cycles):
            e.upload()
            out.append(e.allocate())
        e.close()
    finally:
        for k in opts:
            gpu.debug_option(k, 0)
    return out


def _same(got, ref, what):
    assert np.array_equal(got.visits, ref.visits), f"{what}: visits differ"
    for f in ("task", "node", "kind", "visit"):
        assert len(got.decisions) == len(ref.decisions) and np.array_equal(got.decisions[f], ref.decisions[f]), \
            f"{what}: decision {f} differs"
    assert np.array_equal(got.decisions["score"].view(np.int64), ref.decisions["score"].view(np.int64)), \
        f"{what}: fp64 scores differ"
    assert np.array_equal(got.fit_errors, ref.fit_errors), f"{what}: fit errors differ"


def _counts(res):
    full, reent, rows, past = res.stats["group_reentry"]
    assert res.stats["commit_kernel"] == 1, res.stats  # VC_KERNEL_INCREMENTAL
    assert full + reent == res.stats["prof_cycles"][6], res.stats
    assert rows >= 0 and past >= 0
    return full, reent, rows, past


CASES = {
    # many CTAs (32 nodes each), one queue: groups recur across jobs, a few rows per CTA change in between
    "plain": ("mid_fut", dict(releasing_frac=0.0), {}),
    # Releasing resources: rows move between the idle and the future-idle category while their group is away
    "fut": ("mid_fut", {}, {}),
    # a nearly full cluster: gangs that do not fit are discarded, their rows rolled back, the group re-entered
    "discard": ("mid_fut", dict(releasing_frac=0.0, utilisation=0.97, min_util=0.85), {}),
    # feasible-node sampling windows (SAMP instance)
    "samp": ("mid_fut", dict(releasing_frac=0.0), {"samp": 30}),
    # one CTA holds every node: every placement dirties a row of the only CTA
    "one_cta": ("small", dict(n_nodes=200, n_tasks=3000, n_queues=1, plugins="priority+gang+predicates+nodeorder+binpack"),
                {"VC_COMMIT_CTAS": 1}),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_reentry_matches_oracle(gpu, oracle_engine, name):
    base, changes, opts = CASES[name]
    snap = _snap(base, **changes)
    opts = dict(opts)
    if "samp" in opts:
        snap.conf.percentage_nodes_to_find = opts.pop("samp")
    ref = oracle_engine(snap)
    (res,) = _run(gpu, snap, opts)
    _same(res, ref, name)
    full, reent, rows, past = _counts(res)
    assert reent > 0, (name, res.stats["group_reentry"])
    assert full > 0  # first appearances of the groups
    if name == "discard":
        assert (ref.visits["outcome"] == 2).any(), "no discarded statement: the case does not exercise the rollback"
    if name == "one_cta":
        assert rows > 0 and past <= reent


def test_repeated_cycles_on_one_engine(gpu, oracle_engine):
    """The table is not cleared between cycles: a second and third cycle must not take a stale entry."""
    snap = _snap("mid_fut", releasing_frac=0.0)
    ref = oracle_engine(snap)
    runs = _run(gpu, snap, cycles=3)
    for k, r in enumerate(runs):
        _same(r, ref, f"cycle {k}")
        assert r.stats["group_reentry"] == runs[0].stats["group_reentry"], k


def test_over_budget_session_keeps_full_sweeps(gpu, oracle_engine):
    """Heterogeneous requests: n_groups x node slots x 9 B is over the budget, so every group switch takes a full sweep."""
    snap = _snap("cfg2", n_tasks=12_000, hetero=200)
    slots = -(-snap.N // 128) * 128  # 10k nodes: 79 CTAs x 128 node slots
    key = np.concatenate([snap.t_klass[None, :].astype(np.float64), snap.t_resreq, snap.t_k8s_req,
                          snap.t_k8s_nonzero_req[:2]]).T
    n_groups = len(np.unique(key, axis=0))
    assert n_groups * slots * 9 > VT_BUDGET, n_groups
    res = _run(gpu, snap)[0]
    _same(res, oracle_engine(snap), "over budget")
    full, reent, rows, past = _counts(res)
    assert full > 0 and reent == 0 and rows == 0 and past == 0, res.stats["group_reentry"]
