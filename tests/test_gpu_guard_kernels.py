"""The GUARD instances of the preempt / reclaim kernels (sessions where the pdb or cdp plugin votes) launched on their own
through tools/kernels/evict_harness.cu, production geometry:
  k_evict_rank<16, R, false, true>  the candidate flags against a numpy restatement of the filter, the necessary victim
                                    condition (the last voter of each tier, pdb and cdp among them) and the fit test, from
                                    1 to 200 000 nodes (grid tails included), preempt, intra-job preempt and reclaim;
  k_evict_dryrun<SAMP, true>        ok / nv / victims / the four pick keys against the exact restatement of
                                    SelectVictimsOnNode (tests/topo_kernels_common.py), with ssn.Preemptable's answer
                                    computed here from an independent walk of the pdb budgets (a dict per call) and the
                                    cdp times; nodes of up to 300 pods under many overlapping PDBs, without and with the
                                    sampled list."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import topo_kernels_common as K
from tests.test_gpu_evict_kernels import INTRA, PREEMPT, RECLAIM, RankArgs, _ptr, _rank_case
from volcano_b200 import abi

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(os.path.dirname(HERE), "tools", "kernels", "_build", "evict_harness.so")
NO_LABELS, PDB_NEVER, CDP = 1, 2, 4  # VCT_GUARD_* (vc_topo.hpp)
PDB, CDP_PL = abi.VC_PLUGIN_PDB, abi.VC_PLUGIN_CDP


class EhGuardArgs(C.Structure):
    _fields_ = [("n_pdb", C.c_int), ("bits", C.c_void_p), ("pdb_off", C.c_void_p), ("pdb", C.c_void_p),
                ("pdb_allowed", C.c_void_p)]


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build() compiles it")
    L = C.CDLL(LIB)
    L.eh_rank_guard.argtypes = [C.POINTER(RankArgs), C.c_void_p]
    L.eh_dryrun_guard.argtypes = [C.POINTER(K.EhTopoArgs), C.POINTER(EhGuardArgs), C.c_void_p, C.c_int]
    return L


# ---- rank -------------------------------------------------------------------------------------------------------------
def _guard_rank_case(seed, N, R, tpn, mode):
    a = _rank_case(seed, N, R, tpn, True, mode)
    a["quota_on"] = 0
    rng = np.random.default_rng(seed + 17)
    pl, tiers, en = list(a["plugin"]), list(a["tier"]), list(a["enabled"])
    for g in (PDB, CDP_PL):  # at a random place, often the last voter of its tier
        if rng.random() < 0.85:
            i = int(rng.integers(0, len(pl) + 1))
            t = tiers[i - 1] if i > 0 else 0
            pl.insert(i, g); tiers.insert(i, t)
            en.insert(i, int(rng.choice([abi.VC_EN_PREEMPTABLE | abi.VC_EN_RECLAIMABLE, abi.VC_EN_PREEMPTABLE,
                                         abi.VC_EN_RECLAIMABLE])))
    if seed % 3 == 0:  # one case in three: one tier whose last voter is a guard, in both actions
        pl.append(int(rng.choice([PDB, CDP_PL]))); tiers = [0] * len(pl)
        en.append(abi.VC_EN_PREEMPTABLE | abi.VC_EN_RECLAIMABLE)
    a.update(plugin=np.array(pl, np.int32), tier=np.array(tiers, np.int32), enabled=np.array(en, np.uint32))
    RT = a["RT"]
    bits = np.where(rng.random(RT) < 0.1, NO_LABELS | PDB_NEVER, 0)
    bits |= np.where(rng.random(RT) < 0.3, PDB_NEVER, 0)
    bits |= np.where(rng.random(RT) < 0.3, CDP, 0)
    return a, bits.astype(np.uint8)


def _rank_ref(a, bits):
    """numpy restatement of k_evict_rank's flags (integer requests: the sums are exact in float64)."""
    N, R, RT, mode = a["N"], a["R"], a["RT"], a["mode"]
    pods = a["rt_idx"].astype(np.int64)
    node = np.repeat(np.arange(N), np.diff(a["rt_off"]))
    f, j = a["rt_flags"][pods].astype(np.int64), a["rt_job"][pods].astype(np.int64)
    jj = np.maximum(j, 0)
    q = np.where(j >= 0, a["j_queue"][jj], -1)
    qq = np.maximum(q, 0)
    keep = (a["rt_evicted"][pods] == 0) & (f & abi.VC_RT_PREEMPTABLE != 0)
    if mode == RECLAIM:
        keep &= (f & abi.VC_RT_RUNNING != 0) & (j >= 0) & (q >= 0) & (q != a["queue"]) & \
            (a["q_flags"][qq] & abi.VC_QUEUE_NOT_RECLAIMABLE == 0)
    else:
        keep &= f & (abi.VC_RT_RUNNING | abi.VC_RT_BOUND) != 0
        keep &= (j == a["job"]) if mode == INTRA else ((j >= 0) & (j != a["job"]) & (q == a["queue"]))
    reclaim = mode == RECLAIM
    flag = abi.VC_EN_RECLAIMABLE if reclaim else abi.VC_EN_PREEMPTABLE
    last = {}
    for pl, tier, e in zip(a["plugin"], a["tier"], a["enabled"]):
        if not e & flag:
            continue
        if pl == abi.VC_PLUGIN_CONFORMANCE:
            v = f & abi.VC_RT_CRITICAL == 0
        elif pl == abi.VC_PLUGIN_GANG:
            v = (j >= 0) & (a["j_ready"][jj] > a["j_min"][jj])
        elif pl == abi.VC_PLUGIN_PRIORITY and not reclaim:
            v = (j >= 0) & np.where(j != a["job"], a["j_prio"][jj] < a["job_prio"], a["rt_prio"][pods] < a["task_prio"])
        elif pl == abi.VC_PLUGIN_DRF and not reclaim:
            v = j >= 0
        elif pl == abi.VC_PLUGIN_PROPORTION and reclaim:
            v = (j >= 0) & (q >= 0) & (a["q_over"][qq] != 0)
        elif pl == PDB:
            v = bits[pods] & PDB_NEVER == 0
        elif pl == CDP_PL:
            v = bits[pods] & CDP == 0
        else:
            continue
        last[int(tier)] = v
    may = np.zeros(RT, bool)
    for v in last.values():
        may |= v
    n_pass = np.bincount(node[keep], minlength=N)
    m = keep & may
    fits = (a["cstat"] & 1) != 0
    for d in range(R):
        if d >= 2 and not a["has"] >> d & 1:
            continue
        freed = np.bincount(node[m], weights=a["rt_req"][d][pods[m]], minlength=N)
        have = ((a["idle"][d] + a["rel"][d]) - a["pip"][d]) + freed
        rq = float(a["req"][d])
        fits &= (rq < have) | (np.abs(rq - have) < 0.1)
    if mode == RECLAIM:
        fits &= n_pass > 0
    return fits.astype(np.uint8)


def _run(H, a, bits):
    N = a["N"]
    cand, key = np.full(N, 77, np.uint8), np.full(N, 7, np.uint64)
    keep = {k: np.ascontiguousarray(v) for k, v in a.items() if isinstance(v, np.ndarray)}
    s = RankArgs()
    for name, _ in RankArgs._fields_:
        if name in keep:
            setattr(s, name, _ptr(keep[name]))
        elif name == "n_plugins":
            s.n_plugins = len(a["plugin"])
        elif name not in ("cand", "key"):
            setattr(s, name, int(a[name]))
    s.cand, s.key = _ptr(cand), _ptr(key)
    return H.eh_rank_guard(C.byref(s), _ptr(bits)), cand


@pytest.mark.parametrize("N,R,tpn", [(1, 3, (5,)), (17, 9, (0, 1, 17)), (1000, 2, (0, 3, 33)), (4099, 12, (1, 16, 40)),
                                     (65_537, 4, (0, 2, 9)), (200_000, 8, (0, 1, 5, 17)), (200_000, 16, (3, 12))])
@pytest.mark.parametrize("mode", [PREEMPT, INTRA, RECLAIM])
def test_rank_guard_flags_vs_numpy(H, N, R, tpn, mode):
    """Not vacuous: over the seeds both outcomes occur, and (intra-job preempt and reclaim) clearing every guard bit changes
    some flag."""
    changed = cands = 0
    for seed in range(3):
        a, bits = _guard_rank_case(5000 * R + 31 * mode + seed + N, N, R, tpn, mode)
        rc, cand = _run(H, a, bits)
        assert rc == 0
        want = _rank_ref(a, bits)
        assert np.array_equal(cand, want), (seed, np.flatnonzero(cand != want)[:10])
        cands += int(want.sum())
        changed += int((_rank_ref(a, np.zeros_like(bits)) != want).any())
    if N >= 1000:
        assert 0 < cands < 3 * N
        assert changed > 0 or mode == PREEMPT  # inter-job preempt: the few same-queue victims rarely decide a node here


def test_rank_guard_rejects_bad_bits(H):
    a, bits = _guard_rank_case(3, 20, 3, (2,), PREEMPT)
    bits[0] = 8
    assert _run(H, a, bits)[0] == -1


# ---- dry run ------------------------------------------------------------------------------------------------------------
def _guard_dry_case(seed, N, R, n_pdb, heavy):
    rng = np.random.default_rng(seed)
    I = K.random_instance(rng, N, R, max_pods=300, heavy=heavy)
    I.update(sim_state=1, q_exists=1, sim_alloc=0)
    # the instance's voters keep their job-order enables only; pdb and cdp vote, in one of the tier layouts
    base_pl = [int(p) for p in I["plugin"]]
    base_en = [int(e) & ~abi.VC_EN_PREEMPTABLE for e in I["enabled"]]
    layout = [[[PDB], [CDP_PL]], [[PDB, CDP_PL]], [[CDP_PL, PDB]], [[PDB]], [[CDP_PL]], [[CDP_PL], [PDB]]][seed % 6]
    pl, tier, en = list(base_pl), [0] * len(base_pl), list(base_en)
    for t, voters in enumerate(layout):
        for v in voters:
            pl.append(v); tier.append(t); en.append(abi.VC_EN_PREEMPTABLE)
    I.update(plugin=np.array(pl, np.int32), tier=np.array(tier, np.int32), enabled=np.array(en, np.uint32), n_plugins=len(pl))
    RT = I["RT"]
    labelled = rng.random(RT) < 0.9
    pool = max(1, n_pdb // 4)
    lists = []
    for r in range(RT):  # overlapping PDBs: every task draws from a few PDBs of a shared pool
        k = int(rng.integers(0, 5)) if labelled[r] else 0
        base = int(rng.integers(0, n_pdb - pool + 1))
        lists.append(sorted(set(int(x) for x in rng.integers(base, base + pool, k))))
    off = np.zeros(RT + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in lists])
    pdb = np.array([x for lst in lists for x in lst], np.int32)
    allowed = rng.integers(0, 40, n_pdb).astype(np.int32)
    allowed[rng.random(n_pdb) < 0.2] = 0
    now = int(I["now_ns"])
    until = np.where(rng.random(RT) < 0.3, now + rng.integers(-3, 4, RT) * 10 ** 9, abi.VC_COOLDOWN_NONE)
    bits = np.where(labelled, 0, NO_LABELS | PDB_NEVER)
    for r in range(RT):
        if any(allowed[x] <= 0 for x in lists[r]):
            bits[r] |= PDB_NEVER
    bits = (bits | np.where((until != abi.VC_COOLDOWN_NONE) & (until > now), CDP, 0)).astype(np.uint8)
    G = dict(n_pdb=n_pdb, bits=bits, pdb_off=off, pdb=pdb if len(pdb) else np.zeros(1, np.int32), allowed=allowed,
             lists=lists, labelled=labelled, until=until, layout=layout)
    return I, G


def _preemptable(I, G, n):
    """ssn.Preemptable with pdb and cdp on node n's candidates (session_plugins.go:211-259, pdb.go:65-126, cdp.go:75-104)."""
    def keep(r):
        f = int(I["rt_flags"][r])
        if I["rt_evicted"][r] or not f & abi.VC_RT_PREEMPTABLE or not f & (abi.VC_RT_RUNNING | abi.VC_RT_BOUND):
            return False
        j = int(I["rt_job"][r])
        return j == I["job"] if I["intra"] else (j >= 0 and j != I["job"] and I["j_queue"][j] == I["queue"])
    cands = [int(I["rt_idx"][x]) for x in range(I["rt_off"][n], I["rt_off"][n + 1]) if keep(int(I["rt_idx"][x]))]

    def pdb_vote():
        budget, out = {}, []
        for r in cands:
            if not G["labelled"][r]:
                continue
            violated = False
            for p in G["lists"][r]:
                budget[p] = budget.get(p, int(G["allowed"][p])) - 1
                violated |= budget[p] < 0
            if not violated:
                out.append(r)
        return out
    now = int(I["now_ns"])
    for voters in G["layout"]:
        victims = None
        for v in voters:
            c = pdb_vote() if v == PDB else [r for r in cands if not (G["until"][r] != abi.VC_COOLDOWN_NONE and G["until"][r] > now)]
            if not c:
                victims = None
                break
            victims = c if victims is None else ([x for x in victims if x in c] or None)
        if victims is not None:
            return victims
    return []


def _as_conformance(I, G):
    """The instance with pdb and cdp replaced by one conformance voter whose answer on every node is _preemptable's: the
    restatement of the rest of SelectVictimsOnNode then applies unchanged."""
    J = dict(I)
    pl = [int(p) for p in I["plugin"] if p not in (PDB, CDP_PL)]
    en = [int(e) for p, e in zip(I["plugin"], I["enabled"]) if p not in (PDB, CDP_PL)]
    J.update(plugin=np.array(pl + [abi.VC_PLUGIN_CONFORMANCE], np.int32), tier=np.zeros(len(pl) + 1, np.int32),
             enabled=np.array(en + [abi.VC_EN_PREEMPTABLE], np.uint32), n_plugins=len(pl) + 1)
    fl = I["rt_flags"] | np.uint32(abi.VC_RT_CRITICAL)
    for n in range(I["N"]):
        for r in _preemptable(I, G, n):
            fl[r] &= ~np.uint32(abi.VC_RT_CRITICAL)
    J["rt_flags"] = fl
    return J


def _launch(H, I, G, samp_list):
    a, out = K.to_args(I)
    g = EhGuardArgs(G["n_pdb"], _ptr(G["bits"]), _ptr(G["pdb_off"]), _ptr(G["pdb"]), _ptr(G["allowed"]))
    lst = None if samp_list is None else np.ascontiguousarray(samp_list, np.int32)
    rc = H.eh_dryrun_guard(C.byref(a), C.byref(g), None if lst is None else _ptr(lst), 0 if lst is None else len(lst))
    return rc, out


@pytest.mark.parametrize("N,R,n_pdb,heavy,seed", [(1, 2, 8, 1, 0), (7, 5, 64, 3, 1), (129, 9, 200, 6, 2), (1000, 4, 512, 8, 3),
                                                  (1000, 16, 64, 8, 4), (20_000, 3, 2000, 12, 5)])
@pytest.mark.parametrize("samp", [False, True])
def test_dryrun_guard_matches_the_restatement(H, N, R, n_pdb, heavy, seed, samp):
    """Every node up to 1 000 nodes; beyond, 1 500 sampled nodes plus every node running more than 100 pods. Under SAMP
    the kernel runs on a shuffled half of the predicate nodes only; the other nodes stay untouched."""
    I, G = _guard_dry_case(900 + seed, N, R, n_pdb, heavy)
    rng = np.random.default_rng(seed)
    samp_list = None
    if samp:
        pred = np.flatnonzero(I["pred"])
        samp_list = rng.permutation(pred)[: max(1, len(pred) // 2) if len(pred) else 0]
    rc, out = _launch(H, I, G, samp_list)
    assert rc == 0
    ref = _as_conformance(I, G)
    pods = np.diff(I["rt_off"])
    if samp:
        listed = np.zeros(N, bool)
        listed[samp_list] = True
        assert not out["ok"][:N][~listed].any()
        nodes = samp_list if len(samp_list) <= 1500 else np.union1d(rng.choice(samp_list, 1500, replace=False),
                                                                     np.intersect1d(samp_list, np.flatnonzero(pods > 100)))
    else:
        nodes = np.arange(N) if N <= 1000 else np.union1d(rng.choice(N, 1500, replace=False), np.flatnonzero(pods > 100))
    hits = K.check_dry_run(ref, out, nodes)
    assert N < 100 or hits > 0
    if N >= 129:  # the guards decide: with them off (every pod a victim of both) some node's outcome differs
        G2 = dict(G, labelled=np.ones(I["RT"], bool), allowed=np.full(n_pdb, 10 ** 6, np.int32),
                  until=np.full(I["RT"], abi.VC_COOLDOWN_NONE))
        heavy_nodes = [int(n) for n in nodes if pods[n] > 100][:4] or [int(n) for n in nodes[:50]]
        assert any(_preemptable(I, G, n) != _preemptable(I, G2, n) for n in heavy_nodes)


def test_dryrun_guard_rejects_bad_tables(H):
    I, G = _guard_dry_case(5, 10, 3, 8, 1)
    G["pdb"] = G["pdb"].copy()
    if I["RT"] and G["pdb_off"][-1] > 0:
        G["pdb"][0] = G["n_pdb"]
        assert _launch(H, I, G, None)[0] == -1
    I, G = _guard_dry_case(5, 10, 3, 8, 1)
    assert _launch(H, I, G, np.array([10], np.int32))[0] == -1
