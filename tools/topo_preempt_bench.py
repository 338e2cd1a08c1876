"""Topology-aware preemption on the cfg5 cycle (BASELINE.json configs[4] distribution, allocate + preempt + reclaim):
time vc_preempt_run with enableTopologyAwarePreemption on the state allocate left, end to end (host clock around the
call, which ends with the device idle) and on the device (the two dry-run kernels' share, from the host time spent
waiting for their hand-out), against the normal reading on the same session and the topology-aware oracle
(tools/topo_oracle, one host thread: its dry runs are a sequential loop). The statements of the timed GPU run are compared
with the oracle's. Prints the card's name and power limit read in the same run, then one JSON line.
usage: python tools/topo_preempt_bench.py [n_nodes] [n_pending] [repeats]   (run on the GPU box)"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from volcano_b200 import engine  # noqa: E402
from volcano_b200.snapshot import PreemptArguments  # noqa: E402
from volcano_b200.synth import make_cfg5  # noqa: E402

n_nodes = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000
n_pending = int(sys.argv[2]) if len(sys.argv) > 2 else 1_500
repeats = int(sys.argv[3]) if len(sys.argv) > 3 else 2
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
engine.init(0)


def session(topo):
    snap = make_cfg5(seed=77, n_nodes=n_nodes, n_pending=n_pending, n_queues=8, utilisation=0.9)
    if topo:
        snap.preempt_args = PreemptArguments(topology_aware=True)
        snap.preempt_seed, snap.now_ns = 12345, 7 * 10 ** 9
    return snap


def run(topo):
    """-> (preempt ms end to end, ms waiting for hand-outs, kernel launches, result) of the best of `repeats`."""
    best = None
    for _ in range(repeats):
        e = engine.Engine(session(topo))
        e.upload()
        e.allocate()
        t0 = time.perf_counter()
        rp = e.preempt()
        ms = 1e3 * (time.perf_counter() - t0)
        e.close()
        row = (ms, rp.stats["prof_cycles"][1] / 1e3, rp.stats["kernel_launches"], rp)
        if best is None or ms < best[0]:
            best = row
    return best


topo = run(True)
normal = run(False)
from tests import topo_common as X  # noqa: E402

o = X.TopoOracle(session(True))
o.allocate()
u0 = time.perf_counter()
op = o.preempt()
cpu_ms = 1e3 * (time.perf_counter() - u0)
o.close()
same = np.array_equal(topo[3].visits, op.visits) and all(
    np.array_equal(topo[3].decisions[f], op.decisions[f]) for f in ("task", "node", "kind", "visit"))
print(card)
print(json.dumps({
    "workload": f"cfg5: {n_nodes} nodes at 90 % utilisation, {n_pending} pending tasks, 8 queues; preempt after allocate",
    "card": card, "topology_aware_preempt_ms": topo[0], "topology_aware_waiting_for_device_ms": topo[1],
    "topology_aware_launches": topo[2], "topology_aware_evictions": int((topo[3].decisions["kind"] == 2).sum()),
    "normal_preempt_ms": normal[0], "normal_launches": normal[2],
    "oracle_topology_aware_preempt_ms_1_thread": cpu_ms, "statements_identical_to_oracle": bool(same)}))
