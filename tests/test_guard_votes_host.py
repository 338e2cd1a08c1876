"""The library's own pdb and cdp votes on the CPU (tests/hostshim/guard_shim.cpp, g++): the host vote of
vch::EvictSession (preempt's normal reading, reclaim) and the dry run's vct::topo_vote<true> on the bits the library
stages for the device. The reference's plugin tests transcribed onto them, and random tables against the guard oracle's
plain restatement."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import guard_common as G
from tests.test_guard_evict_cpu import LABEL, _vote_session
from volcano_b200 import abi
from volcano_b200.api import BuildPDB, BuildPod, BuildResourceList

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostshim", "guard_shim.cpp")
OUT = os.path.join(HERE, "hostshim", "_build", "guard_shim.so")


@pytest.fixture(scope="module")
def S():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", SRC, "-o", OUT], check=True)
    L = C.CDLL(OUT)
    L.gs_votes.argtypes = [C.c_int, C.POINTER(abi.vc_victim_guards), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L


def _votes(S, plugin, snap, cands):
    vg = snap.victim_guards()
    c = np.array(cands, np.int32)
    host, dev = np.zeros(max(len(c), 1), np.uint8), np.zeros(max(len(c), 1), np.uint8)
    assert S.gs_votes(plugin, C.byref(vg), c.ctypes.data, len(c), host.ctypes.data, dev.ctypes.data) == 0
    return [int(r) for r, y in zip(c, host) if y], [int(r) for r, y in zip(c, dev) if y]


@pytest.mark.parametrize("pdbs,want", [
    ([], [0, 1]),
    ([BuildPDB("default", "test-pdb", {LABEL: "job-1"}, 0)], []),
    ([BuildPDB("default", "test-pdb", {LABEL: "job-1"}, 1)], [0]),
])
def test_pdb_preemptable_and_reclaimable_fn(S, pdbs, want):
    """plugins/pdb/pdb_test.go TestPreemptableAndReclaimableFn on the library's votes."""
    pods = [BuildPod("default", f"test-pod{i + 1}", "n0", "Running", BuildResourceList("1", "1G"), "pg", {LABEL: "job-1"})
            for i in range(2)]
    assert _votes(S, abi.VC_PLUGIN_PDB, _vote_session(pods, pdbs, "pdb"), [0, 1]) == (want, want)


def test_cdp_preemptable_fn(S):
    """plugins/cdp/cdp_test.go TestPreemptableFn on the library's votes: task1 kept, task2 and task3 victims."""
    now = 10 ** 18
    pods = []
    for name, cool, ago in (("t1", "600s", 100), ("t2", "600abcde", 100), ("t3", "600s", 800)):
        p = BuildPod("default", name, "n0", "Running", BuildResourceList("1", "1G"), "pg", {"volcano.sh/preemptable": "true"})
        p.annotations = {"volcano.sh/cooldown-time": cool}
        p.scheduled_time = now - ago * 10 ** 9
        pods.append(p)
    assert _votes(S, abi.VC_PLUGIN_CDP, _vote_session(pods, [], "cdp", now), [0, 1, 2]) == ([1, 2], [1, 2])


def test_random_tables_match_the_oracle(S):
    """Random tables (budgets 0-3, overlapping selectors, unlabelled pods, DisruptedPods, cooldowns on both sides of now,
    until == now included) and random candidate lists: host vote, dry-run vote and the oracle's plain walk agree."""
    rng = np.random.default_rng(7)
    differ = 0
    for trial in range(150):
        n = int(rng.integers(1, 40))
        now = 10 ** 18
        pods = []
        for i in range(n):
            labels = {}
            if rng.random() < 0.85:
                labels["app"] = str(rng.choice(["a", "b"]))
                if rng.random() < 0.5:
                    labels["tier"] = str(rng.choice(["x", "y"]))
            p = BuildPod("default", f"p{i}", "n0", "Running", BuildResourceList("1", "1G"), "pg", labels)
            if rng.random() < 0.4:
                p.annotations = {"volcano.sh/cooldown-time": "100s"}
                p.scheduled_time = now - int(rng.integers(98, 103)) * 10 ** 9
            pods.append(p)
        sels = [{"app": "a"}, {"app": "b"}, {"tier": "x"}, {"app": "a", "tier": "y"}, {}]
        pdbs = [BuildPDB("default", f"b{k}", sels[int(rng.integers(0, len(sels)))], int(rng.integers(0, 4)),
                         [f"p{i}" for i in range(n) if rng.random() < 0.1]) for k in range(int(rng.integers(0, 5)))]
        cands = sorted(int(x) for x in rng.choice(n, int(rng.integers(0, n + 1)), replace=False))
        for plugin, name in ((abi.VC_PLUGIN_PDB, "pdb"), (abi.VC_PLUGIN_CDP, "cdp")):
            snap = _vote_session(pods, pdbs, name, now)
            host, dev = _votes(S, plugin, snap, cands)
            o = G.GuardOracle(snap)
            try:
                want = o.vote(plugin, cands)
            finally:
                o.close()
            assert host == want and dev == want, (trial, name, cands, host, dev, want)
            differ += want != cands
    assert differ > 50
