"""Topology-aware preemption on the H100: vc_preempt_run with vc_preempt_options against the topology-aware oracle
(tools/topo_oracle) and the upstream expectations, and the option switched off against no option at all."""
import importlib.util
import os

import numpy as np
import pytest

from tests import topo_common as X
from tests.golden import topo_preempt_cases as G
from volcano_b200.snapshot import PreemptArguments

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gpu():
    from volcano_b200 import engine
    engine.init(0)
    return engine


def _fuzz():
    spec = importlib.util.spec_from_file_location("fuzz_evict", os.path.join(ROOT, "tools", "fuzz_evict.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("case", G.golden_cases(), ids=lambda c: c.Name[:50])
def test_goldens_through_vc_preempt_run(gpu, case):
    case.RegisterSession(G.topo_tiers(), actions=("preempt",), configurations=G.TOPO, preempt_seed=1, now_ns=0)
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()


@pytest.mark.parametrize("case", G.golden_cases(), ids=lambda c: c.Name[:50])
def test_goldens_through_the_action(gpu, case):
    """test.Run([preempt.New()]) as the reference's test drives it."""
    from volcano_b200 import preempt
    case.RegisterSession(G.topo_tiers(), actions=("preempt",), configurations=G.TOPO, preempt_seed=1, now_ns=0)
    case.Run([preempt.New("preempt")])
    assert case.CheckAll() is None, case.CheckAll()


@pytest.mark.parametrize("case,tiers,kw", X.hand_cases(), ids=lambda c: getattr(c, "Name", "")[:50])
def test_hand_derived(gpu, case, tiers, kw):
    case.RegisterSession(tiers, actions=("preempt",), **kw)
    case.Run(gpu.gpu_engine)
    assert case.CheckAll() is None, case.CheckAll()


@pytest.mark.parametrize("block", range(6))
def test_topo_family_matches_the_oracle(gpu, block):
    """tools/fuzz_evict.py's topo family, 40 sessions per block: allocate / preempt / reclaim chains with the option on,
    proportion with and without EnabledPredicate, varied seeds, clocks and candidate counts. Every statement identical."""
    F = _fuzz()
    ran = 0
    for seed in range(block * 40, block * 40 + 40):
        tc, tiers, actions, conf = F.make_topo_case(seed)
        snap = tc.RegisterSession(tiers, actions=actions, **conf)
        if snap.T == 0 or snap.N == 0 or snap.B > 0:
            continue
        try:
            ref = X.oracle_engine(snap)
        except RuntimeError:  # outside the path (refused by both): the library must refuse too
            with pytest.raises(gpu.VcError):
                gpu.gpu_engine(snap)
            continue
        F.compare(gpu.gpu_engine(snap), ref, seed)
        ran += 1
    assert ran >= 30


@pytest.mark.parametrize("block", range(2))
def test_option_off_is_byte_identical(gpu, block):
    """The options set with topology_aware = 0 give exactly what no options give."""
    F = _fuzz()
    for seed in range(block * 30, block * 30 + 30):
        tc, tiers, actions = F.make_case(seed)
        plain = tc.RegisterSession(tiers, actions=actions)
        if plain.T == 0 or plain.N == 0 or plain.B > 0:
            continue
        try:
            a = gpu.gpu_engine(plain)
        except gpu.VcError:
            continue
        off = tc.RegisterSession(tiers, actions=actions, configurations={"preempt": {"enableTopologyAwarePreemption": False,
                                                                                    "minCandidateNodesAbsolute": 3}})
        assert off.preempt_args is not None and not off.preempt_args.topology_aware
        b = gpu.gpu_engine(off)
        assert np.array_equal(a.decisions, b.decisions) and np.array_equal(a.visits, b.visits), seed
        for name in ("preempt", "reclaim"):
            x, y = getattr(a, name), getattr(b, name)
            assert (x is None) == (y is None)
            if x is not None:
                assert x.decisions.tobytes() == y.decisions.tobytes() and x.visits.tobytes() == y.visits.tobytes(), (seed, name)


@pytest.mark.parametrize("n_nodes", [1000, 10_000])
def test_cfg5_cycle_with_topology_aware_preemption(gpu, n_nodes):
    """BASELINE configs[4] (nodes near capacity, ~1 500 pending tasks, 8 queues): allocate -> preempt -> reclaim with the
    option on, every statement against the oracle."""
    from volcano_b200.synth import make_cfg5
    snap = make_cfg5(seed=77, n_nodes=n_nodes, n_pending=1500, n_queues=8, utilisation=0.9)
    snap.preempt_args = PreemptArguments(topology_aware=True)
    snap.preempt_seed, snap.now_ns = 12345, 7 * 10 ** 9
    rng = np.random.default_rng(3)
    snap.rt_pod_priority = rng.integers(0, 3, snap.RT).astype(np.int32)
    snap.rt_start_ns = np.where(rng.random(snap.RT) < 0.2, np.iinfo(np.int64).min,
                                rng.integers(0, 5, snap.RT) * 10 ** 9).astype(np.int64)
    res = gpu.gpu_engine(snap)
    ref = X.oracle_engine(snap)
    _fuzz().compare(res, ref, n_nodes)
    assert (ref.preempt.decisions["kind"] == 2).sum() > 10
