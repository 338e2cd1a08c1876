"""Preempt and reclaim under the reference's default feasible-node sampling (adaptive percentage, min-nodes-to-find 100,
5 % at 10 000 nodes) on a cfg5 cycle: allocate -> preempt -> reclaim on the GPU for the normal and the topology-aware
reading of preempt, then the same actions on the sampling oracle (one host thread) with every statement compared.
Prints one JSON line with the card's name and power limit.
usage: python tools/samp_evict_bench.py [seed] [n_nodes] [n_pending]   (run on the GPU box)"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import samp_common as S  # noqa: E402
from volcano_b200 import engine  # noqa: E402
from volcano_b200.snapshot import PreemptArguments  # noqa: E402
from volcano_b200.synth import make_cfg5  # noqa: E402

seed = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
n_nodes = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
n_pending = int(sys.argv[3]) if len(sys.argv) > 3 else 10_000


def session(topo):
    snap = make_cfg5(seed=seed, n_nodes=n_nodes, n_pending=n_pending)
    snap.conf.percentage_nodes_to_find, snap.conf.min_nodes_to_find, snap.conf.min_percentage_nodes_to_find = 0, 100, 5
    snap.conf.enable_predicate_error_cache = 0
    if topo:
        snap.preempt_args = PreemptArguments(topology_aware=True)
        snap.preempt_seed, snap.now_ns = 12345, 10 ** 9
    return snap


engine.init(0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
out = {"gpu": gpu, "nodes": n_nodes, "pending": n_pending}
same = True
for name, topo in (("normal", False), ("topology_aware", True)):
    snap = session(topo)
    e = engine.Engine(snap)
    try:
        e.upload()
        res = e.allocate()
        t0 = time.perf_counter()
        res.preempt = e.preempt()
        t1 = time.perf_counter()
        res.reclaim = e.reclaim()
        t2 = time.perf_counter()
    finally:
        e.close()
    o = S.SampOracle(snap)
    try:
        ref = o.allocate()
        t3 = time.perf_counter()
        ref.preempt = o.preempt()
        ref.reclaim = o.reclaim()
        t4 = time.perf_counter()
    finally:
        o.close()
    same = same and S.same(res, ref)
    out[f"{name}_preempt_ms"] = round((t1 - t0) * 1e3, 1)
    out[f"{name}_reclaim_ms"] = round((t2 - t1) * 1e3, 1)
    out[f"{name}_launches"] = res.preempt.stats["kernel_launches"] + res.reclaim.stats["kernel_launches"]
    out[f"{name}_waiting_for_device_ms"] = round((res.preempt.stats["prof_cycles"][1] + res.reclaim.stats["prof_cycles"][1]) / 1e3, 1)
    out[f"{name}_oracle_preempt_reclaim_ms_1_thread"] = round((t4 - t3) * 1e3, 1)
    out[f"{name}_evictions"] = int(sum((r.decisions["kind"] == 2).sum() for r in (res.preempt, res.reclaim)))
out["statements_identical_to_oracle"] = bool(same)
print(json.dumps(out))
