"""Preempt and reclaim on a cfg5 cycle with the network-topology-aware plugin: allocate -> preempt -> reclaim on the GPU,
then the same actions on the oracle extension (tools/nta_evict_oracle, one host thread) with every statement compared.
cfg5's running and pending distribution sits under BASELINE config 4's 3-tier HyperNode tree (32 x 40 leaves, a root and
the cluster top hypernode); the plugin joins cfg5's second tier with config 4's arguments, and a fifth of the jobs that
run pods are soft-mode topology jobs (they reclaim and are victims, they never preempt). Four runs of the same session:
- binpack_on: hypernode binpacking of normal pods on, weight 10;
- binpack_off: binpacking off, so the evicting actions launch the kernels of a session without the term; it evicts
  other pods than binpack_on, so the difference between the two is not the cost of the term alone;
- zero_on / zero_off: the plugin's weight 0 (it scales the soft-mode topology score too, so both differ from the runs
  above), binpacking on / off. zero_on launches the NTA kernels, which compute the term and book the hypernodes' usage
  on every statement, but the term is 0 on every node: its statements must equal zero_off's, and the difference in
  time between the two is the cost of the term alone.
Prints one JSON line with the card's name and power limit, read in the same run.
usage: python tools/nta_evict_bench.py [seed] [n_nodes] [n_pending] [soft_job_percent]   (GPU box)"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import nta_common as NT  # noqa: E402
from tests import samp_common as S  # noqa: E402
from volcano_b200 import engine, synth  # noqa: E402
from volcano_b200.snapshot import build_conf  # noqa: E402

seed = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
n_nodes = int(sys.argv[2]) if len(sys.argv) > 2 else 10_000
n_pending = int(sys.argv[3]) if len(sys.argv) > 3 else 10_000
soft_pct = float(sys.argv[4]) if len(sys.argv) > 4 else 20.0


def session(binpack, weight=10):
    snap = synth.make_cfg5(seed=seed, n_nodes=n_nodes, n_pending=n_pending)
    rng = np.random.default_rng(seed + 23)
    cfg = synth.SynthConfig("cfg5_nta", n_nodes, snap.T, snap.Q, synth.CFG5_PLUGINS + "+network-topology-aware",
                            topology=(32, 40), soft_topology_frac=0.0)
    synth._make_topology(snap, cfg, rng)
    running_jobs = np.unique(snap.rt_job[snap.rt_job >= 0])
    soft = running_jobs[rng.random(len(running_jobs)) < soft_pct / 100.0]
    snap.hn_job_soft[soft] = 1
    sconf = synth.scheduler_conf(cfg)
    sconf.actions = ("allocate", "preempt", "reclaim")
    for t in sconf.tiers:
        for o in t:
            if o.name == "network-topology-aware":
                o.arguments["hypernode.binpack.normal-pod.enable"] = binpack
                o.arguments["weight"] = weight
    snap.conf = build_conf(sconf, synth.DIMS, synth.KDIMS)
    snap.actions = tuple(sconf.actions)
    return snap


engine.init(0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
out = {"gpu": gpu, "nodes": n_nodes, "pending": n_pending, "soft_job_percent": soft_pct}
same = True
results = {}
for name, binpack, weight in (("binpack_on", True, 10), ("binpack_off", False, 10), ("zero_on", True, 0),
                              ("zero_off", False, 0)):
    snap = session(binpack, weight)
    if name == "binpack_on":
        out["soft_jobs"] = int(snap.hn_job_soft.sum())
        out["hypernodes"] = len(snap.hn_names)
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
    same = same and S.same(res, NT.run(snap), index=False)
    results[name] = res
out["statements_identical_to_oracle"] = bool(same)
out["zero_on_statements_identical_to_zero_off"] = bool(S.same(results["zero_on"], results["zero_off"], index=False))
print(json.dumps(out))
