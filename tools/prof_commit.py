"""Phase profile of the commit kernel (cycles of CTA 0) on a synthetic config; run on the GPU box."""
import json
import os
import sys
import time

os.environ.setdefault("VC_PROF", "1")  # the instrumented instance of the incremental kernel

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from volcano_b200 import engine  # noqa: E402
from volcano_b200.synth import make_snapshot  # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
snap = make_snapshot(cfg)
if os.environ.get("SAMP"):  # feasible-node sampling (percentage-nodes-to-find, 0 = the reference's adaptive default)
    snap.conf.percentage_nodes_to_find = int(os.environ["SAMP"]) if os.environ["SAMP"].isdigit() else 0
e = engine.Engine(snap)
e.upload()
for _ in range(2):
    r = e.allocate()
t0 = time.perf_counter()
e.upload()
t1 = time.perf_counter()
r = e.allocate()
t2 = time.perf_counter()
st = r.stats
prof = st["prof_cycles"]
tot = sum(prof[:5]) or 1
names = ["queue/job control", "task fetch+gates", "node sweep", "exchange", "apply+bookkeeping"]
out = {"cfg": cfg, "ctas": os.environ.get("VC_COMMIT_CTAS"), "threads": os.environ.get("VC_COMMIT_THREADS"),
       "commit_ms": st["commit_ms"], "upload_ms": 1e3 * (t1 - t0), "run_ms": 1e3 * (t2 - t1), "steps": st["n_steps"],
       "placed": len(r.decisions), "us_per_step": 1e3 * st["commit_ms"] / max(1, st["n_steps"]),
       "cycles_per_step": tot / max(1, st["n_steps"]),
       "phases": {n: round(p / tot, 3) for n, p in zip(names, prof)},
       "pods_per_s": len(r.decisions) / (st["commit_ms"] * 1e-3), "full_sweeps": prof[6], "incremental": prof[7], "owner_changes": prof[5],
       "group_reentry": st["group_reentry"]}
print(json.dumps(out))
e.close()
