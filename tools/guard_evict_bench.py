"""Preempt and reclaim on a cfg5 cycle with the pdb and cdp plugins: allocate -> preempt -> reclaim on the GPU, then the
same actions on the guard oracle (tools/guard_oracle, one host thread) with every statement compared. PodDisruptionBudgets
cover part of the running jobs (one PDB per job, all its pods, DisruptionsAllowed 0-3), a few running pods carry no labels,
and part of the pods a volcano.sh/cooldown-time whose end lies on either side of now. pdb and cdp join conformance's tier,
so the actions launch the GUARD instances of k_evict_rank. The same session also runs without the two plugins (the
kernels every session launched before); the two evict different pods, so their difference in time is not the cost of the
votes alone. A third run isolates that cost: the same plugins and table shape, but every budget too large to run out,
every pod labelled and every cooldown over, so the votes return every candidate and the statements must equal those of
the run without the plugins. Prints one JSON line with the card's name and power limit, read in the same run.
usage: python tools/guard_evict_bench.py [seed] [n_nodes] [n_pending] [pdb_job_percent] [cooldown_percent]   (GPU box)"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import guard_common as G  # noqa: E402
from tests import samp_common as S  # noqa: E402
from volcano_b200 import abi, engine  # noqa: E402
from volcano_b200.synth import make_cfg5  # noqa: E402

seed = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
n_nodes = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
n_pending = int(sys.argv[3]) if len(sys.argv) > 3 else 10_000
pdb_pct = float(sys.argv[4]) if len(sys.argv) > 4 else 30.0
cool_pct = float(sys.argv[5]) if len(sys.argv) > 5 else 20.0
NOW = 10 ** 18


def session(kind):
    snap = make_cfg5(seed=seed, n_nodes=n_nodes, n_pending=n_pending)
    if kind == "no_guards":
        return snap
    rng = np.random.default_rng(seed + 11)
    c = snap.conf
    tier = next(c.plugins[i].tier for i in range(c.n_plugins) if c.plugins[i].plugin == abi.VC_PLUGIN_CONFORMANCE)
    at = max(i for i in range(c.n_plugins) if c.plugins[i].tier == tier) + 1
    opts = [(c.plugins[i].plugin, c.plugins[i].tier, c.plugins[i].enabled) for i in range(c.n_plugins)]
    opts[at:at] = [(abi.VC_PLUGIN_PDB, tier, abi.VC_EN_ALL), (abi.VC_PLUGIN_CDP, tier, abi.VC_EN_ALL)]
    c.n_plugins = len(opts)
    for i, (pl, t, en) in enumerate(opts):
        c.plugins[i].plugin, c.plugins[i].tier, c.plugins[i].enabled = pl, t, en
    RT = snap.RT
    jobs = np.unique(snap.rt_job[snap.rt_job >= 0])
    covered = jobs[rng.random(len(jobs)) < pdb_pct / 100.0]
    pdb_of = {int(j): i for i, j in enumerate(covered)}
    snap.g_flags = np.where(rng.random(RT) < 0.02, abi.VC_GUARD_NO_LABELS, 0).astype(np.uint32)
    lst, off = [], [0]
    for r in range(RT):
        p = pdb_of.get(int(snap.rt_job[r]), -1)
        if p >= 0 and not snap.g_flags[r]:
            lst.append(p)
        off.append(len(lst))
    snap.g_pdb_off, snap.g_pdb = np.array(off, np.int32), np.array(lst, np.int32)
    snap.g_pdb_allowed = rng.integers(0, 4, len(covered)).astype(np.int32)
    snap.g_until = np.full(RT, abi.VC_COOLDOWN_NONE, np.int64)
    cool = rng.random(RT) < cool_pct / 100.0
    snap.g_until[cool] = NOW + rng.integers(-600, 600, int(cool.sum())) * 10 ** 9
    if kind == "neutral_guards":  # the votes can change nothing: they still run on every candidate list
        snap.g_flags[:] = 0
        lst, off = [], [0]
        for r in range(RT):
            p = pdb_of.get(int(snap.rt_job[r]), -1)
            if p >= 0:
                lst.append(p)
            off.append(len(lst))
        snap.g_pdb_off, snap.g_pdb = np.array(off, np.int32), np.array(lst, np.int32)
        snap.g_pdb_allowed[:] = 10 ** 9
        snap.g_until[cool] = NOW - rng.integers(1, 600, int(cool.sum())) * 10 ** 9
    snap.now_ns = NOW
    return snap


engine.init(0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
out = {"gpu": gpu, "nodes": n_nodes, "pending": n_pending, "pdb_job_percent": pdb_pct, "cooldown_percent": cool_pct}
same = True
results = {}
for name in ("no_guards", "guards", "neutral_guards"):
    snap = session(name)
    if name == "guards":
        out["pdbs"] = int(len(snap.g_pdb_allowed))
    e = engine.Engine(snap)
    try:
        e.upload()
        t0 = time.perf_counter()
        res = e.allocate()
        t1 = time.perf_counter()
        res.preempt = e.preempt()
        t2 = time.perf_counter()
        res.reclaim = e.reclaim()
        t3 = time.perf_counter()
    finally:
        e.close()
    out[f"{name}_allocate_ms"] = round((t1 - t0) * 1e3, 1)
    out[f"{name}_preempt_ms"] = round((t2 - t1) * 1e3, 1)
    out[f"{name}_reclaim_ms"] = round((t3 - t2) * 1e3, 1)
    out[f"{name}_preempt_launches"] = res.preempt.stats["kernel_launches"]
    out[f"{name}_reclaim_launches"] = res.reclaim.stats["kernel_launches"]
    out[f"{name}_evictions"] = int(sum((r.decisions["kind"] == 2).sum() for r in (res.preempt, res.reclaim)))
    print(name, "device path done, oracle comparison running", file=sys.stderr, flush=True)
    same = same and S.same(res, G.run(snap), index=False)
    results[name] = res
out["statements_identical_to_oracle"] = bool(same)
out["neutral_statements_identical_to_no_guards"] = bool(S.same(results["neutral_guards"], results["no_guards"], index=False))
print(json.dumps(out))
