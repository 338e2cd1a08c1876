"""Preempt and reclaim on a cfg5 cycle with PreferNoSchedule taints: allocate -> preempt -> reclaim on the GPU, then the
same actions on the sampling oracle (one host thread) with every statement compared. The taints sit on a few percent of
the nodes (an autoscaler marking scale-down candidates), under nodeorder's default tainttoleration.weight 3, so preempt's
normal reading takes the SOFT instances of its kernels. Each shape also runs without the taints, which launches the
kernels sessions without soft taints always launched; the two sessions evict different pods, so their difference in time
is not the cost of the soft-taint reduction alone. Both without feasible-node sampling and
under the reference's default adaptive sampling (5 % at 10 000 nodes). Prints one JSON line with the card's name and
power limit, read in the same run; statements_identical_to_oracle covers all four runs.
usage: python tools/steady_evict_bench.py [seed] [n_nodes] [n_pending] [tainted_percent]   (run on the GPU box)"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import samp_common as S  # noqa: E402
from volcano_b200 import engine  # noqa: E402
from volcano_b200.synth import make_cfg5  # noqa: E402

seed = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
n_nodes = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
n_pending = int(sys.argv[3]) if len(sys.argv) > 3 else 10_000
tainted_pct = float(sys.argv[4]) if len(sys.argv) > 4 else 3.0


def session(soft, samp):
    snap = make_cfg5(seed=seed, n_nodes=n_nodes, n_pending=n_pending)
    if soft:  # 1-3 PreferNoSchedule taints (of 8 keys) on tainted_pct % of the nodes; no class tolerates them
        rng = np.random.default_rng(seed + 7)
        bits = np.zeros(snap.N, np.uint64)
        for n in np.flatnonzero(rng.random(snap.N) < tainted_pct / 100.0):
            for b in rng.choice(8, int(rng.integers(1, 4)), replace=False):
                bits[n] |= np.uint64(1) << np.uint64(int(b))
        snap.n_taint_soft[0] = bits
        snap.c_tolerated_soft[:] = 0
    if samp:
        snap.conf.percentage_nodes_to_find, snap.conf.min_nodes_to_find, snap.conf.min_percentage_nodes_to_find = 0, 100, 5
        snap.conf.enable_predicate_error_cache = 0
    return snap


engine.init(0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
out = {"gpu": gpu, "nodes": n_nodes, "pending": n_pending, "tainted_percent": tainted_pct}
same = True
for samp in (False, True):
    for soft in (False, True):
        name = ("sampled_" if samp else "all_nodes_") + ("soft" if soft else "no_taints")
        snap = session(soft, samp)
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
        same = same and S.same(res, S.run(snap), index=samp)
out["statements_identical_to_oracle"] = bool(same)
print(json.dumps(out))
