"""Commit-kernel device time of cfg3 with and without hierarchical drf, in one process, alternating.

cfg3_hdrf is cfg3 (10 000 nodes x 100 000 tasks, 16 queues, drf + proportion) with its queues under a 3-level tree:
4 departments x 4 teams, unequal weights. Prints one JSON line with the card's name and power limit read in the same run.
    python tools/hdrf_bench.py [--reps 3] [--generic]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--generic", action="store_true", help="time k_commit (VC_COMMIT_GENERIC=1)")
    args = ap.parse_args()
    from volcano_b200 import engine
    from volcano_b200.synth import make_snapshot
    engine.init(0)
    engine.debug_option("VC_COMMIT_GENERIC", 1 if args.generic else 0)
    flat = make_snapshot("cfg3")
    hd = make_snapshot("cfg3_hdrf")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    times = {"cfg3": [], "cfg3_hdrf": []}
    n_dec = {}
    for _ in range(args.reps + 1):  # the first pair warms up
        for name, snap in (("cfg3", flat), ("cfg3_hdrf", hd)):
            e = engine.Engine(snap)
            e.upload()
            r = e.allocate()
            times[name].append(r.stats["commit_ms"])
            n_dec[name] = len(r.decisions)
            e.close()
    out = {"card": card, "kernel": "general" if args.generic else "incremental",
           "commit_ms": {k: v[1:] for k, v in times.items()}, "decisions": n_dec}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
